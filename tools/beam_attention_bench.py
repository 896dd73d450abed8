"""Cost of the attention export of beam search (decode.beam_decode(..., return_attention=True)) on the cfg #5 workload of
tools/ragged_decode_bench.py: 256 images of height 64, widths 64..1024, seed 5, bf16 storage on the wgmma / mma.sync kernels, beam 5,
the images as one list (every image at its own size in one time loop).  Random-init weights never emit END, so every call runs
max_length_formula + 2 = 152 steps.  decode.beam_decode is timed three ways, each the faster of two timed passes after a warm-up pass:
without attention, with finalize='reference' attention and with finalize='backtrack' attention.  From a separate torch.profiler run
of the backtrack call: lo_beam_backtrack's kernel time against its HBM byte bound, (beam * n * sum_i R_i + n_img * beam * n * R) * 4 B
over 3.35 TB/s (the rows it reads, and the output it writes, padded to the largest region count R).  The card's name, power limit
and max SM clock are read in the same run.

    python tools/beam_attention_bench.py [--out DIR]     (one JSON line on stdout; the profiler table under DIR if given)
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch

import ragged_decode_bench as rdb
from latex_ocr_b200 import decode
from latex_ocr_b200.data import SimpleVocab
from latex_ocr_b200.img2seq import Img2SeqModel

BEAM = 5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for the profiler table")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is nothing to measure on the CPU")
    m = Img2SeqModel(rdb.Cfg(), vocab=SimpleVocab(rdb.V), device="cuda:0", precision="bf16", impl="tc").build_pred()
    m.train_mode(False)
    end_id = m._end_id()
    imgs, _ = rdb.workload()
    out = {"card": rdb.card(),
           "workload": "cfg5: %d images %d x {%s} px as one list, bf16 + tc, beam %d, %d decode steps (random-init weights never emit "
                       "END); host uint8 images in, ids, log-probs and attention on the CPU out; faster of two timed passes after a "
                       "warm-up pass" % (rdb.N_IMG, rdb.HEIGHT, ",".join(map(str, rdb.WIDTHS)), BEAM, rdb.MAX_LEN + 2)}
    call = lambda **kw: decode.beam_decode(m, imgs, end_id - 1, end_id, BEAM, rdb.MAX_LEN, **kw)
    arms = {"off": {}, "reference": {"return_attention": True}, "backtrack": {"finalize": "backtrack", "return_attention": True}}
    res = {}
    for name, kw in arms.items():
        dt, res[name] = rdb.timed(lambda: call(**kw))
        out["beam5_%s_seconds" % name] = dt
        out["beam5_%s_img_s" % name] = rdb.N_IMG / dt
    ids, _, att = res["backtrack"]
    n = ids.shape[2]
    counts = [a.shape[2] for a in att]
    out["steps"] = n
    out["ids_reference_equal_off"] = bool(torch.equal(res["reference"][0], res["off"][0]) and torch.equal(res["reference"][1], res["off"][1]))
    out["attention_bytes_to_host"] = sum(a.numel() for a in res["reference"][2]) * 4
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call(finalize="backtrack", return_attention=True)
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "beam_backtrack_kernel" in e.key]
    if not ev:
        raise SystemExit("profile has no beam_backtrack_kernel")
    dev_us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in ev)
    byts = (BEAM * n * sum(counts) + len(counts) * BEAM * n * max(counts)) * 4
    out["backtrack_kernel_launches"] = sum(e.count for e in ev)
    out["backtrack_kernel_us"] = dev_us
    out["backtrack_kernel_bytes"] = byts
    out["backtrack_kernel_bound_us"] = byts / rdb.HBM_BYTES_PER_S * 1e6
    out["backtrack_kernel_share_of_byte_bound"] = out["backtrack_kernel_bound_us"] / dev_us
    memcpy = [e for e in prof.key_averages() if "Memcpy DtoH" in e.key]
    out["dtoh_copy_us"] = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in memcpy)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "beam_attention_profile.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=25))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
