"""cfg #5 (BASELINE.json configs[4]) decoded three ways on the TensorFlow-flavour model (img2seq_tf, Genthial cell, model.json's
attention sizes): greedy and beam-2 (model.json's beam size) tokens/s and images/s of
  (a) bucketed: one predict_batch call per image shape (no padding inside a shape);
  (b) ragged:   one Img2SeqModel.predict_images call, every image at its own size in one time loop;
  (c) padded:   one predict_batch call, all images padded to the largest (64 x 1024 px).
The images are tools/ragged_decode_bench.py's: 256 images of height 64, widths 64..1024, seed 5, bf16 storage on the wgmma /
mma.sync kernels, host uint8 images in, token ids out; faster of two timed passes after one warm-up pass.  Tokens are counted
after truncation at END.  Also printed: the token agreement of (b) with (a), the agreement of (a) with itself when every shape's
batch is split in two halves (how much the dense path's tokens move with its batch alone), and the card with its power limit.

    python tools/tf_ragged_decode_bench.py     (one JSON line on stdout)
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import torch

from latex_ocr_b200.data import SimpleVocab
from latex_ocr_b200.img2seq_tf import Img2SeqModel
from ragged_decode_bench import HEIGHT, MAX_LEN, N_IMG, V, WIDTHS, card, timed, workload


class Cfg:
    encoder_cnn = "vanilla"; positional_embeddings = True; lr_init = 1e-3; lr_method = "adam"
    attn_cell_config = {"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}
    max_length_formula = MAX_LEN

    def __init__(self, decoding, beam_size):
        self.decoding, self.beam_size = decoding, beam_size


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is nothing to measure on the CPU")
    imgs, batches = workload()
    out = {"card": card(), "workload": "cfg5 on the TF-flavour model: %d images %d x {%s} px, bf16 + tc, host uint8 images in, token "
                                      "ids out, at most %d decode steps; faster of two timed passes after a warm-up pass"
                                      % (N_IMG, HEIGHT, ",".join(map(str, WIDTHS)), MAX_LEN + 2)}
    for mode, decoding, beam in (("greedy", "greedy", 1), ("beam2", "beam_search", 2)):
        torch.manual_seed(0)                      # the same random-init weights in both modes
        m = Img2SeqModel(Cfg(decoding, beam), vocab=SimpleVocab(V), device="cuda:0", precision="bf16", impl="tc").build_pred()
        m.decoder._ws.maxsize = m.encoder._ws.maxsize = 2 * len(WIDTHS) + 8     # every arm's workspaces stay cached

        def bucketed():
            ids = []
            for b in batches:
                ids += m.predict_batch(b)[0]
            return ids

        arms = {"a_bucketed": bucketed, "b_ragged": lambda: m.predict_images(imgs)[0], "c_padded": lambda: m.predict_batch(imgs)[0]}
        res = {}
        for name, fn in arms.items():
            dt, ids = timed(fn)
            res[name] = ids
            toks = sum(len(s) for s in ids)
            out["%s_%s_tok_s" % (mode, name)] = toks / dt
            out["%s_%s_img_s" % (mode, name)] = N_IMG / dt
            out["%s_%s_seconds" % (mode, name)] = dt
        # (a) lists images in bucket order, (b) in input order: both orders are `imgs`' order bucketed by shape
        key = lambda a: (a.shape, a.tobytes())
        a_ids = {}
        pos = 0
        for b in batches:
            for x in b:
                a_ids.setdefault(key(x), []).append(res["a_bucketed"][pos])
                pos += 1
        match = total = 0
        for x, got in zip(imgs, res["b_ragged"]):
            want = a_ids[key(x)].pop(0)
            match += sum(int(g == w) for g, w in zip(got, want))
            total += max(len(got), len(want))
        out["%s_token_agreement_b_vs_a" % mode] = match / max(total, 1)
        # the same control for the dense path alone: (a) again with every shape's batch split in two halves.  The per-step GEMMs
        # change kernel with the row count, so bf16 sums and near-tie argmaxes change with the batch as well
        halves = []
        for b in batches:
            h = len(b) // 2
            halves += (m.predict_batch(b[:h])[0] if h else []) + m.predict_batch(b[h:])[0]
        match = total = 0
        for got, want in zip(halves, res["a_bucketed"]):
            match += sum(int(g == w) for g, w in zip(got, want))
            total += max(len(got), len(want))
        out["%s_token_agreement_a_halves_vs_a" % mode] = match / max(total, 1)
        out["%s_tokens_b" % mode] = sum(len(s) for s in res["b_ragged"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
