"""Times the TensorFlow-flavour decoder (Genthial cell) forward + loss + backward at the cfg #2 shape (B=64, R=868, T=150,
V=500, bf16) and its greedy / beam-2 decode on one H100.  Prints one JSON line."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from util import Cfg  # noqa: E402
from latex_ocr_b200.tf_decoder import Decoder  # noqa: E402


def timeit(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    B, R, T, V = 64, 868, 150, 500
    cfg = Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=150,
              decoding="greedy")
    g = torch.Generator().manual_seed(0)
    enc = (torch.relu(torch.randn(B, R, 512, generator=g)) * 0.5).cuda()
    formula = torch.randint(0, V, (B, T), generator=g).cuda()
    lengths = torch.randint(20, T + 1, (B,), generator=g)
    dec = Decoder(cfg, V, V - 1, device="cuda", precision="bf16", impl="tc")
    out = {"shape": {"B": B, "R": R, "T": T, "V": V}}
    out["train_fwd_bwd_ms"] = timeit(lambda: dec.loss_and_backward(enc, formula, lengths), 5)
    out["train_fwd_ms"] = timeit(lambda: dec.run_forward(enc, formula, lengths), 5)
    ms = timeit(lambda: dec.decode(enc, max_steps=152), 3)
    out["greedy_152_steps_ms"] = ms
    out["greedy_tokens_per_s"] = B * 152 / (ms * 1e-3)
    cfg2 = Cfg(attn_cell_config=cfg.attn_cell_config, max_length_formula=150, decoding="beam_search", beam_size=2)
    decb = Decoder(cfg2, V, V - 1, device="cuda", precision="bf16", impl="tc")
    ms = timeit(lambda: decb.decode(enc, max_steps=152), 3)
    out["beam2_152_steps_ms"] = ms
    out["loss"] = float(dec.loss_and_backward(enc, formula, lengths)[0][0])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
