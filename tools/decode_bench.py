"""cfg #5 (BASELINE.json): greedy and beam-5 decoding throughput, 256 images of height 64 bucketed by width
{64,128,256,512,1024} (same-shape batches like model/utils/data_generator.py:84-122), random-init weights, bf16.
Random weights never emit END, so every batch runs the full max_length_formula + 2 = 152 steps."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from latex_ocr_b200 import decode
from latex_ocr_b200.data import SimpleVocab
from latex_ocr_b200.img2seq import Img2SeqModel


class Cfg:
    encoder_cnn = "vanilla"; positional_embeddings = True; lr_init = 1e-3; lr_method = "adam"


V = 500
m = Img2SeqModel(Cfg(), vocab=SimpleVocab(V), device="cuda:0", precision="bf16", impl="tc").build_pred()
m.train_mode(False)
g = torch.Generator().manual_seed(0)
buckets = [64, 128, 256, 512, 1024]
per = 256 // len(buckets)
out = {}
for mode, beam in (("greedy", 1), ("beam5", 5)):
    toks, secs = 0, 0.0
    for W in buckets:
        n = per + (1 if W == 1024 else 0)
        img = torch.where(torch.rand(n, 1, 64, W, generator=g) < 0.1, torch.randint(0, 255, (n, 1, 64, W), generator=g).float(), torch.tensor(255.0))
        for rep in range(2):          # first pass warms workspaces
            torch.cuda.synchronize(); t0 = time.perf_counter()
            if beam == 1:
                ids = decode.greedy_decode(m, img, V - 2, V - 1, 150)
                nt = ids.numel()
            else:
                ids, _ = decode.beam_decode(m, img, V - 2, V - 1, beam, 150)
                nt = ids.shape[0] * ids.shape[2]            # tokens of the scored hypothesis
            torch.cuda.synchronize(); dt = time.perf_counter() - t0
        toks += nt; secs += dt
    out[mode] = {"tokens_per_s": toks / secs, "images_per_s": 256 / secs, "seconds": secs}
print(json.dumps({"workload": "cfg5: 256 images 64 x {64..1024}, 152 steps, bf16, 1 x H100", **out}))
