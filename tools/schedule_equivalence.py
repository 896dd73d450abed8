"""Checks that two builds of the library run the decoder's schedules alike: the same number of kernel launches and the same
numbers, case by case, at the cfg #2 shapes (bf16 on the wgmma / mma.sync kernels, B = 64, 128x512 images, V = 500, T = 150).

  python tools/schedule_equivalence.py --base _C_parent [--head _C]

--base / --head name library directories under latex_ocr_b200/ (LO_LIB_DIR of `python -m latex_ocr_b200.build`), e.g. a build of
the parent commit made in another checkout and copied next to this one.  Each run is a process of its own with the library
option "deterministic" = 1; the base build runs twice, which measures the spread of the order-dependent paths, then the head build
runs once.  Every case starts from the same seeded weights and inputs.  Cases:
  torch flavour, one train step (forward, loss, backward, Adam): the default, each of the schedule options dec_streams=2, dec_fuse,
    dec_fuse_bwd, dec_cl, dec_cl_bwd, fuse_lstm, skinny_mma=0, att_pipe=0, scheduled sampling (p = 0.25) and self-critical
    training (tau = 1);
  TensorFlow flavour, one train step: teacher forcing, scheduled sampling, self-critical training;
  both flavours: greedy decode of images of different sizes in one batch (ragged), beam search with the diversity penalty, greedy
    decode of one batch with its attention weights, and beam search of a ragged batch (the TF flavour's with its log-probs).
Compared per case: lo_launch_count() over the case, and the loss, the gradients, the fed tokens and the decoded ids / attention
weights / log-probs.
Launch counts must be equal, and every output bit-identical across the three runs, except on the paths that still add with fp32
atomics under "deterministic".  Those are two torch-flavour paths that DESIGN.md §4 lists: the fused backward step kernels
(dec_fuse_bwd), and the wgmma split-K of the per-step backward GEMMs (skinny_mma=0 puts it on every step).  The third is the
TensorFlow-flavour train step, whose attention backward adds d beta with atomics.  On those paths a head-against-base difference
of up to 1e-4 of the largest magnitude passes.  The base build's difference from itself is printed beside it.  Measured on an H100
80GB HBM3 at a 700 W power limit, that spread was 1e-5 to 3e-5 of max-abs on the two torch paths and below 1e-7 on the TF step.
Prints one line per case and exits non-zero on a mismatch.
"""
import argparse
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, H, W, T, V = 64, 128, 512, 150, 500
OPTION_CASES = {"default": {}, "dec_streams=2": {"dec_streams": 2}, "dec_fuse": {"dec_fuse": 1}, "dec_fuse_bwd": {"dec_fuse_bwd": 1},
                "dec_cl": {"dec_cl": 1}, "dec_cl_bwd": {"dec_cl_bwd": 1}, "fuse_lstm": {"fuse_lstm": 1}, "skinny_mma=0": {"skinny_mma": 0},
                "att_pipe=0": {"att_pipe": 0}}
ORDER_DEPENDENT = {"dec_fuse_bwd", "skinny_mma=0", "tf_default", "tf_sampling", "tf_scst"}
TOL = 1e-4
DECODE_WIDTHS = (128, 192, 256, 320, 384, 448, 512, 160, 224, 288, 352, 416, 480, 512, 128, 256)
BEAM, DIV_GAMMA, DIV_PROB = 5, 0.5, 0.5


def run_cases():
    """Child process: every case on the build LO_LIB_DIR selects -> {case: (launches, {name: CPU tensor})}."""
    sys.path.insert(0, ROOT)
    import torch
    import bench_support as bs
    from latex_ocr_b200 import _lib, decode
    from latex_ocr_b200.data import SimpleVocab
    from latex_ocr_b200.img2seq import Img2SeqModel
    from latex_ocr_b200.img2seq_tf import Img2SeqModel as TfModel

    _lib.set_option("deterministic", 1)

    class Cfg:
        encoder_cnn = "vanilla"; positional_embeddings = True; lr_init = 1e-3; lr_method = "adam"; cuda_graph = False

    class TfCfg:
        attn_cell_config = {"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}
        max_length_formula = T; lr_init = 1e-3; lr_method = "adam"; clip = -1; dropout = 1.0

        def __init__(self, decoding="greedy"):
            self.decoding, self.beam_size, self.div_gamma, self.div_prob = decoding, BEAM, DIV_GAMMA, DIV_PROB

    def torch_model():
        torch.manual_seed(1234)
        m = Img2SeqModel(Cfg(), vocab=SimpleVocab(V), device="cuda", precision="bf16", impl="tc")
        m.build_train()
        m.train_mode(True)
        return m

    def tf_model(decoding="greedy"):
        torch.manual_seed(1234)
        return TfModel(TfCfg(decoding), vocab=SimpleVocab(V), device="cuda", precision="bf16", impl="tc").build_train()

    img, formula = bs.synthetic_batch(B, H, W, V, T, seed=1234)
    img, formula = img.cuda(), formula.cuda()
    tf_img, tf_formula = bs.synthetic_batch(B, H, W, V, T - 1, seed=1234)          # T columns: tokens, END, PAD
    tf_img, tf_formula = tf_img.to(torch.uint8).cuda(), tf_formula.cuda()
    tf_lengths = (tf_formula != V - 2).sum(dim=1).to(torch.int32)
    ragged = [img[i, :, :, :w].to(torch.uint8).cpu().contiguous() for i, w in enumerate(DECODE_WIDTHS)]
    dense = img[:len(DECODE_WIDTHS)].to(torch.uint8)
    res = {}

    def record(name, fn):
        torch.cuda.synchronize()
        l0 = _lib.launch_count()
        out = fn()
        torch.cuda.synchronize()
        res[name] = (_lib.launch_count() - l0, {k: v.detach().cpu().clone() for k, v in out.items()})
        print("  %s: %d launches" % (name, res[name][0]), flush=True)

    def train(m, step, fed=False):
        def fn():
            loss = step()
            out = {"loss": loss, "grad_decoder": m.decoder.store.grad, "grad_encoder": m.encoder.store.grad}
            if fed:
                out["fed"] = m.decoder.last_fed_tokens
            return out
        return fn

    for name, opts in OPTION_CASES.items():
        with _lib.option(**opts):
            m = torch_model()
            record(name, train(m, lambda: m.train_step(img, formula)))
    m = torch_model()
    m.set_sampling_prob(0.25)
    record("sampling", train(m, lambda: m.train_step(img, formula), fed=True))
    m = torch_model()
    m.set_self_critical(1.0)
    record("scst", train(m, lambda: m.train_step(img, formula), fed=True))
    m = torch_model()
    end_id = m._end_id()
    record("greedy_ragged", lambda: {"ids": decode.greedy_decode(m, ragged, end_id - 1, end_id, T)})
    m = torch_model()

    def beam():
        ids, logp = decode.beam_decode(m, dense, end_id - 1, end_id, BEAM, T, div_gamma=DIV_GAMMA, div_prob=DIV_PROB, div_seed=7)
        return {"ids": ids, "logp": logp}
    record("beam_div", beam)
    m = torch_model()

    def greedy_att():
        ids, alphas = decode.greedy_decode(m, dense, end_id - 1, end_id, T, return_attention=True)
        return {"ids": ids, "alphas": alphas}
    record("greedy_att", greedy_att)
    m = torch_model()

    def beam_ragged():
        ids, logp = decode.beam_decode(m, ragged, end_id - 1, end_id, BEAM, T)
        return {"ids": ids, "logp": logp}
    record("beam_ragged", beam_ragged)

    tf_step = lambda m: (lambda: m.train_step(tf_img, (tf_formula.cpu(), tf_lengths.cpu())))
    m = tf_model()
    record("tf_default", train(m, tf_step(m)))
    m = tf_model()
    m.set_sampling_prob(0.25)
    record("tf_sampling", train(m, tf_step(m), fed=True))
    m = tf_model()
    m.set_self_critical(1.0)
    record("tf_scst", train(m, tf_step(m), fed=True))
    m = tf_model()
    record("tf_greedy_ragged", lambda: {"ids": torch.tensor([t for s in m.predict_images(ragged)[0] for t in s + [-1]])})
    m = tf_model("beam_search")
    record("tf_beam_div", lambda: {"ids": torch.tensor([t for h in m.predict_batch(dense) for s in h for t in s + [-1]])})
    m = tf_model()

    def tf_greedy_att():
        out, alphas = m.decoder.decode(m.encoder.forward_raw(dense), return_attention=True)
        return {"ids": out.ids, "alphas": alphas}
    record("tf_greedy_att", tf_greedy_att)
    m = tf_model("beam_search")

    def tf_beam_ragged():
        encs = [m.encoder.forward_raw(x[None].cuda())[0].clone() for x in ragged]     # each run overwrites the encoder's output
        out, logp = m.decoder.decode(encs, return_log_probs=True)
        return {"ids": out.ids, "logp": logp}
    record("tf_beam_ragged", tf_beam_ragged)
    return res


def rel_diff(a, b):
    """max |a - b| over max |a|."""
    ref = a.double().abs().max().item()
    return (a.double() - b.double()).abs().max().item() / (ref or 1.0)


def compare(base, again, head):
    """base, again: two runs of the base build (the spread of an order-dependent path); head: the build under test."""
    import torch
    bad = 0
    for case, (n0, out0) in base.items():
        n1, out1 = head[case]
        tol = case in ORDER_DEPENDENT
        notes, failed = [], n0 != n1 or again[case][0] != n0
        if failed:
            notes.append("launches %d (base again %d) vs %d" % (n0, again[case][0], n1))
        for k, a in out0.items():
            b, a2 = out1[k], again[case][1][k]
            if a.shape != b.shape or a.dtype != b.dtype:
                failed = True
                notes.append("%s: shape/dtype %s %s vs %s %s" % (k, tuple(a.shape), a.dtype, tuple(b.shape), b.dtype))
                continue
            if torch.equal(a, b) and torch.equal(a, a2):
                continue
            if tol and a.is_floating_point():
                d, spread = rel_diff(a, b), rel_diff(a, a2)
                failed |= d > TOL
                notes.append("%s: %.1e of max-abs (base against itself %.1e)" % (k, d, spread))
            else:
                failed = True
                notes.append("%s: %d of %d elements differ (base against itself: %d)" % (k, int((a != b).sum()), a.numel(),
                                                                                        int((a != a2).sum())))
        bad += failed
        print("%-18s %-8s launches %6d  %s" % (case, "MISMATCH" if failed else "ok", n0, "; ".join(notes) or "bit-identical"))
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="library directory under latex_ocr_b200/ of the build compared against")
    ap.add_argument("--head", default="_C", help="library directory under latex_ocr_b200/ of the build under test")
    ap.add_argument("--child", metavar="FILE", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        import torch
        torch.save(run_cases(), args.child)
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    res = []
    with tempfile.TemporaryDirectory() as tmp:
        for i, tag in enumerate((args.base, args.base, args.head)):
            path = os.path.join(tmp, "%d.pt" % i)
            print("build %s:" % tag, flush=True)
            subprocess.run([sys.executable, os.path.abspath(__file__), "--base", args.base, "--child", path], check=True,
                           env=dict(os.environ, LO_LIB_DIR=tag))
            res.append(torch.load(path))
    bad = compare(*res)
    print("%d of %d cases match" % (len(res[0]) - bad, len(res[0])))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
