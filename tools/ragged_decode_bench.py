"""cfg #5 (BASELINE.json configs[4]) decoded three ways: greedy and beam-5 tokens/s and images/s of
  (a) bucketed: one decode per image shape, as bench_support.decode_probe times it;
  (b) ragged:   one Img2SeqModel.predict_images call, every image at its own size in one time loop;
  (c) padded:   one predict_batch call, all images padded to the largest (64 x 1024 px).
The workload is decode_probe's: 256 images of height 64, widths 64..1024, seed 5, bf16 storage on the wgmma / mma.sync kernels,
host uint8 images in, token ids out; faster of two timed passes after one warm-up pass.  Random-init weights never emit END, so
every arm runs max_length_formula + 2 = 152 steps.  Also printed: the token agreement of (b) with (a), and, from a separate
torch.profiler run of (b), the ragged attention kernel's time per step against its HBM byte bound.

    python tools/ragged_decode_bench.py [--out DIR]     (one JSON line on stdout; the profiler table under DIR if given)
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from latex_ocr_b200 import data as lod
from latex_ocr_b200.data import SimpleVocab
from latex_ocr_b200.img2seq import Img2SeqModel

V, N_IMG, HEIGHT, WIDTHS, MAX_LEN = 500, 256, 64, (64, 128, 256, 512, 1024), 150
HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


class Cfg:
    encoder_cnn = "vanilla"; positional_embeddings = True; lr_init = 1e-3; lr_method = "adam"


def workload():
    """decode_probe's images (same generator, same order) and its same-shape batches"""
    rng = np.random.RandomState(5)
    per = N_IMG // len(WIDTHS)
    imgs = []
    for i, W in enumerate(WIDTHS):
        n = per + (N_IMG - per * len(WIDTHS) if i == len(WIDTHS) - 1 else 0)
        for _ in range(n):
            a = np.full((HEIGHT, W, 1), 255, np.uint8)
            ink = rng.rand(HEIGHT, W, 1) < 0.10
            a[ink] = rng.randint(0, 255, size=int(ink.sum())).astype(np.uint8)
            imgs.append(a)
    order = rng.permutation(len(imgs))
    items = lod.bucket_by_shape([(imgs[i], int(i)) for i in order], per)
    batches = [[it[0] for it in items[k:k + per]] for k in range(0, len(items), per)]
    return [imgs[i] for i in order], [b for b in batches if b]


def timed(fn):
    """(seconds of the faster of two timed passes after a warm-up pass, the result of the last pass)"""
    best, out = None, None
    for rep in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        if rep > 0:
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
    return best, out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for the profiler table")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is nothing to measure on the CPU")
    m = Img2SeqModel(Cfg(), vocab=SimpleVocab(V), device="cuda:0", precision="bf16", impl="tc").build_pred()
    m.train_mode(False)
    m.decoder._ws.maxsize = m.encoder._ws.maxsize = 2 * len(WIDTHS) + 8     # every arm's workspaces stay cached
    cfg = m._config
    cfg.max_length_formula = MAX_LEN
    imgs, batches = workload()
    out = {"card": card(), "workload": "cfg5: %d images %d x {%s} px, bf16 + tc, host uint8 images in, token ids out, %d decode steps "
                                      "(random-init weights never emit END); faster of two timed passes after a warm-up pass"
                                      % (N_IMG, HEIGHT, ",".join(map(str, WIDTHS)), MAX_LEN + 2)}
    for mode, beam in (("greedy", 1), ("beam5", 5)):
        cfg.decoding = "greedy" if beam == 1 else "beam_search"
        cfg.beam_size = beam

        def bucketed():
            ids = []
            for b in batches:
                ids += m._decode_ids(torch.from_numpy(lod.pad_batch_images(b)).permute(0, 3, 1, 2).contiguous())[0][0]
            return ids

        arms = {"a_bucketed": bucketed, "b_ragged": lambda: m.predict_images(imgs)[0], "c_padded": lambda: m.predict_batch(imgs)[0]}
        res = {}
        for name, fn in arms.items():
            dt, ids = timed(fn)
            res[name] = ids
            toks = sum(len(s.split()) if isinstance(s, str) else len(s) for s in ids)
            out["%s_%s_tok_s" % (mode, name)] = toks / dt
            out["%s_%s_img_s" % (mode, name)] = N_IMG / dt
            out["%s_%s_seconds" % (mode, name)] = dt
        # (a) lists images in bucket order, (b) and (c) in input order: both orders are `imgs`' order bucketed by shape
        key = lambda a: (a.shape, a.tobytes())
        a_ids = {}
        pos = 0
        for b in batches:
            for x in b:
                a_ids.setdefault(key(x), []).append(res["a_bucketed"][pos])
                pos += 1
        match = total = 0
        for x, got in zip(imgs, m._decode_ids(list(imgs))[0][0]):          # (b)'s ids before truncation and formatting
            want = a_ids[key(x)].pop(0)
            match += sum(int(g == w) for g, w in zip(got, want))
            total += max(len(got), len(want))
        out["%s_token_agreement_b_vs_a" % mode] = match / max(total, 1)
    # ragged attention kernel time per step vs its byte bound (separate, profiled run of arm (b), greedy)
    cfg.decoding, cfg.beam_size = "greedy", 1
    from torch.profiler import ProfilerActivity, profile
    m.predict_images(imgs)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.predict_images(imgs)
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "attention_fwd_ragged_kernel" in e.key]
    if not ev:
        raise SystemExit("profile has no ragged attention kernel")
    dev_us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in ev)
    calls = sum(e.count for e in ev)
    counts = []
    for x in imgs:
        h, w = m.encoder.out_hw(x.shape[0], x.shape[1])
        counts.append(h * w)
    A = C = 512
    step_bytes = sum(r * (A + C) * 2 + r * 4 for r in counts)          # att1 + enc rows (bf16) read, alphas written (fp32)
    per_step_us = dev_us / calls
    out["attention_ragged_us_per_step"] = per_step_us
    out["attention_ragged_launches"] = calls
    out["attention_ragged_bytes_per_step"] = step_bytes
    out["attention_ragged_bound_us"] = step_bytes / HBM_BYTES_PER_S * 1e6
    out["attention_ragged_share_of_byte_bound"] = (step_bytes / HBM_BYTES_PER_S * 1e6) / per_step_us
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ragged_decode_profile.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=25))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
