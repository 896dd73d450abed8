"""Balanced-bracket decode (decode.BracketRule, the *_brackets entry points) against the same decode without the rule, on cfg #5
(BASELINE.json configs[4]): the 256 images of tools/ragged_decode_bench.py (height 64, widths 64..1024, host uint8 images in one
list), V = 500, bf16 storage on the wgmma / mma.sync kernels, 152 steps (random-init weights never emit END).  Modes: greedy,
beam 5 with finalize='backtrack', and sample 8 (tau 1, no filter).  The rule is the LaTeX rule of a synthetic vocabulary with
``{`` / ``}``, ``\\left(`` / ``\\right)`` and ``\\begin{array}`` / ``\\end{array}`` (three kinds, max_depth 16): its cost does not
depend on which tokens carry roles, one bracket_mask_kernel launch per step reading the role table and writing the excluded
logits.

The six arms (mode x rule off / on) alternate inside one process: a warm-up pass of each, then five rounds in which every arm
runs once, each pass timed with CUDA events around the call.  Reported per arm: the fastest and the slowest pass in ms, and per
mode the ratio on / off of the fastest passes.  The card's name, power limit and maximum SM clock, read in the same process, are
printed beside the numbers.

    python tools/bracket_decode_bench.py     (one JSON line on stdout)
"""
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

START, END = rdb.V - 2, rdb.V - 1
BEAM, N_S, ROUNDS = 5, 8, 5
BRACKETS = {10: "{", 11: "}", 12: "\\left(", 13: "\\right)", 14: "\\begin{array}", 15: "\\end{array}"}


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is nothing to measure on the CPU")
    m = Img2SeqModel(rdb.Cfg(), vocab=SimpleVocab(rdb.V), device="cuda:0", precision="bf16", impl="tc").build_pred()
    m.train_mode(False)
    imgs, _ = rdb.workload()
    rule = decode.BracketRule.latex([BRACKETS.get(i, "t%d" % i) for i in range(rdb.V)])
    modes = {
        "greedy": lambda br: decode.greedy_decode(m, imgs, START, END, rdb.MAX_LEN, brackets=br),
        "beam5": lambda br: decode.beam_decode(m, imgs, START, END, BEAM, rdb.MAX_LEN, finalize="backtrack", brackets=br)[0],
        "sample8": lambda br: decode.sample_decode(m, imgs, START, END, N_S, max_length_formula=rdb.MAX_LEN, seed=1, brackets=br)[0],
    }
    arms = [(mode, on) for mode in modes for on in (False, True)]

    def run(mode, on):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        ids = modes[mode](rule if on else None)
        e1.record()
        torch.cuda.synchronize()
        if on:
            assert all(rule.check(ids, END))
        return e0.elapsed_time(e1)

    out = {"card": rdb.card(),
           "workload": "cfg5: %d images %d x {%s} px in one list, V %d, bf16 + tc, %d decode steps; greedy, beam %d (backtrack), "
                       "sample %d (tau 1); LaTeX bracket rule (3 kinds, max_depth 16) off / on alternating, %d rounds after a "
                       "warm-up, CUDA events" % (rdb.N_IMG, rdb.HEIGHT, ",".join(map(str, rdb.WIDTHS)), rdb.V, rdb.MAX_LEN + 2,
                                                 BEAM, N_S, ROUNDS)}
    for a in arms:
        run(*a)
    times = {a: [] for a in arms}
    for _ in range(ROUNDS):
        for a in arms:
            times[a].append(run(*a))
    for mode in modes:
        off, on = times[(mode, False)], times[(mode, True)]
        out[mode] = {"off_ms": [round(min(off), 2), round(max(off), 2)], "on_ms": [round(min(on), 2), round(max(on), 2)],
                     "ratio_on_off": round(min(on) / min(off), 4)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
