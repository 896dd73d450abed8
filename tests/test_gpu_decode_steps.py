"""-m gpu: the decode loops (greedy_loop, sample_loop and beam_loop of csrc/lo_decoder.cu) step by step against float64
(tests/decode_step_ref.py, tests/decoder_step_ref.py, tests/tfdec_step_ref.py), through all nine entry points:
lo_decoder_{greedy_hist,beam_pen,sample} (torch flavour), lo_decoder2_{greedy,beam,sample} (the two-layer decoder of the
extension) and lo_tfdec_{greedy,beam_pen,sample} (TensorFlow flavour), under the schedules a decode reads: the per-step GEMMs
(skinny_mma, skinny_tma, skinny8), PDL, the attention forward (att_pipe, att_nsplit, att_cluster, att_l2_keep_mb) and
deterministic.  The other options (att_maskbits, att_bwd_mma, wgrad256, conv_mc, ...) are read by training paths only.

Getting step t's operands.  A decode keeps only the current step's logits, finished flags, parent rows, lengths and coverage, and
the beam reorder overwrites hall[t+1] / call[t+1] in place.  So each case runs the same call with max_steps = 1 .. T from
sentinel-filled buffers (and the same Philox state) and snapshots the buffers after each.  That relies on decode being
deterministic, which is asserted: every shorter call's outputs (tokens or ids / parents / fin_hist) and the per-step buffers it
wrote (hall, call, out1, alphas, ctx, gctx, gates) are a bit-for-bit prefix of the longer call's.

Checks, from the operands each launch read (bounds of tests/test_gpu_decoder_steps.py, through tests/step_check.py):
  * the prologue: row b's mean is image b // rows_per_img's mean over its own regions ((R_i + 1) 2^-24 sum |enc| / R_i), h0 and
    c0 within (2^-16 + 2^-18) S on the tensor-core path (the hi + lo bf16 halves of the mean), 2^-16 S otherwise.
  * each step: out1 (GEMM rule), alphas / ctx / gctx (the 1e-5 rule) with row b attending over its own image's rows only, the
    entries of alphas past an image's region count keep the sentinel (the ragged kernel writes [0, R_i) only), the gates
    (Lipschitz allowances) from the token the row was fed (the start token at t = 0), c and h from the kernel's own gates.
  * beam reorder: hall[t+1][b] / call[t+1][b] are the cell of row parent_rows[b] (its stored gates and the c it read) within the
    cell bounds; slots with the same parent are bit-identical; on the tensor-core path the bf16 mirror of hall[t+1] is
    RN_bf16(hall[t+1]) bit for bit (the recast after the gather).
  * logits: fc(RN(h)) (tensor cores) or fc(h) within 2^-16 S for every row in greedy and sampling decode.  In beam search the h
    from before the gather survives only for rows that are some slot's parent, and those rows' logits are checked against it;
    the other rows' logits come from the same GEMM launch over h the cell check covered, and they enter every decision through
    the log-softmax the decision check below evaluates on the kernel's own logits.
  * choices, on the kernel's own fp32 logits: the greedy argmax exactly (the lowest index among equals).  In beam search and
    sampling each candidate's key gets an fp32 allowance: the log-softmax ((V + 8) 2^-24 + 2^-23 |lse| + 2^-24 |lp|, the rule of
    the cross-entropy check), one rounding per add, the length division and the coverage add (2^-24 of the result each), the
    diversity rank times |log gamma| for every other candidate of the row whose total lies within the two allowances, and for
    the Gumbel score 2^-22 (|x / tau| + |log(-log u)| + 1) (the division, logf of the uniform, logf of that).  Where two
    candidates' float64 keys differ by more than their allowances added, the kernel's order must be the float64 order; within
    that, either order is accepted (and counted); candidates computed from the same fp32 inputs (ties built from duplicate
    fc.weight rows, or fc.weight = 0 with repeated bias values) tie bit for bit in the kernel too and must come in the documented
    order, the lower flat index first.  fin_hist, next_tok, parent_rows and len_out must follow from the chosen candidates as
    integers; logp and scores must be their float64 totals and keys within the allowances; the coverage within one rounding
    (2^-24 of itself) and its term within (2^-16 + 2^-22) of its magnitude sum.  The sampled token must lie in the kept set, its
    top-p cut taken anywhere the mass before a position is within (V + 10) 2^-23 of itself from top_p, and must win the draw over
    every token surely kept.  A finished row costs END 0 and every other token -FLT_MAX in beam search; in sampling it emits END
    and adds nothing; in greedy decode it keeps emitting its argmax (the reference's greedy cell decodes on; the caller
    truncates).
  * the two-layer decoder (cases l2_*): layer 1 as above; layer 2 from the slot it read (the zero state at t = 0), its gates from
    h1 and that h2, c2 and h2 from its own gates, the bf16 mirror of h2, the logits fc(h2) of every row.  In beam search step t
    writes slot 1 (h2 before the gather, so the logits of every row are checked) and the reorder gathers it into slot 0, the slot
    the next step reads: h2, c2 and the mirror by parent_rows bit for bit.
  * the TF flavour (cases tf_*), from its workspace (tests/tfdec_step_ref.py carve) with the bounds of
    tests/test_gpu_tfdec_steps.py: att_img per image, the token table, each row's own image mean, initpre and the initial state
    (copied bit for bit into xh[0] and call[0]); per step the gates from xh[t] and the token fed (row V, the start token, at
    t = 0), c and h from the kernel's own gates, out2, the attention over the row's own image (the tanh.approx rule on the tensor
    cores), ctx and its bf16 mirror, o, and the logits.  The reorder (xh with its mirror, then c): xh[t+1] and call[t+1] are the
    cell of row parent_rows[b], slots of one parent bit-identical, xh_bf[t+1] is RN_bf16(xh[t+1]) bit for bit; out2 and the
    logits are checked on the parent rows, whose state the gather kept.  Then every choice by the rules above.

Cases: fp32 and bf16 on the CUDA cores, bf16 on the tensor cores; 4 to 1,025 rows (head_nt on mma.sync up to 64 rows, gemm_nt
above); greedy; beam 1, 3, 5 and 16 (16 x V = 500 with a penalty takes the > 48 kB shared-memory path), with alpha, beta, both,
and the diversity penalty with injected and Philox uniforms; sampling with 1 and 8 samples per image, top_k = 1, 5, 20 and V, a
top_p that keeps one token, a top_p on an exact boundary (all logits equal: the masses i / V are exact, and the token right past
the cut gets the largest uniform), top_p = 0.8 / 0.9 / 0.95, tau = 0.5 and 2, V = 501 (not a multiple of the four Philox words)
and V = 2048 (8 sort positions per thread); rows finishing at different steps through fc.bias[END]; a ragged list of 3 to 44
regions; 205 images x beam 5; the bench's decode shape (51 images of
372 regions, the encoder's 6 x 62 for 64 x 512 px, beam 5, bf16 on tensor cores).

Worst |y - ref| / bound per quantity, over every case and schedule, measured on an H100 80GB HBM3 (700 W power limit); the whole
file (78 runs) ran in 37 s there:
    roundings of one value (a value next to a rounding midpoint nears the bound): att1 (bf16) 0.986, coverage 0.9998; TF
        att_img (bf16) 0.983
    pointwise: c 0.463, h 0.433, gates 0.026, out1 gate 0.033; TF c 0.482, h 0.460, gates 0.022, sinit 0.221, o 0.009
    log-softmax rule: beam logp 0.051, beam scores 0.083, sample logp 0.045 (TF flavour 0.025, 0.057, 0.040)
    attention: alphas 0.023, ctx 0.030, gctx 0.006 (1e-5 rule); TF alphas 0.002, ctx 0.001 (tanh.approx rule)
    GEMMs and reductions (2^-16 S): out1 att2 0.017, out1 hh 0.019, mean 0.46, h0 c0 0.035, logits 0.017, coverage term 0.010;
        TF mean 0.47, initpre 0.015, ptab 0.013, out2 0.015, logits 0.016
    decisions inside the fp32 margin (accepted either way): 13 in b5_1025, 6 in b5_pen_ragged, 3 in b5_bench, 1-2 in five
        other beam cases; 72 / 13 / 5 / 2 rows whose top-p cut lies within the margin in s8_V2048, s8_p09_ragged, tf_s8, s8_V501
        (their tokens still checked against the surely kept set)
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import decode_step_ref as dr
import decoder_step_ref as ds
from step_check import ACC, SENTINEL, ULPS, Checker, bits, check_cell, check_gates, rn

pytestmark = pytest.mark.gpu

_E = 512
START = 1
END = 3

# name: dict(mode, precision, impl, images: N x R or a list of region counts, rpi, T, V, and the mode's settings)
#   ties "dup": fc rows 10..19 copies of row 10 with the largest bias (exact ties); "zero": fc.weight = 0 and bias values
#   repeated (every row's logits tie in groups); "const": every logit equal, so the top-p masses are exact and top_p = 0.25 falls
#   on a position (u_peak: that token's uniform the largest); end_bias: fc.bias[END] (rows finish at different steps)
_RAGGED = [44, 20, 7, 31, 12, 44, 25, 3]
_CASES = {
    "g_fp32": dict(mode="greedy", prec="fp32", impl="simt", images=(8, 44), T=6, end_bias=0.5),
    "g_bf16simt": dict(mode="greedy", prec="bf16", impl="simt", images=_RAGGED, T=5, end_bias=0.45),
    "g_tc72": dict(mode="greedy", prec="bf16", impl="tc", images=(72, 40), T=4, end_bias=0.5),
    "g_tc_ragged": dict(mode="greedy", prec="bf16", impl="tc", images=_RAGGED, T=5, end_bias=0.45),
    "g_dup": dict(mode="greedy", prec="bf16", impl="tc", images=(8, 44), T=3, ties="dup"),
    "g_zero": dict(mode="greedy", prec="fp32", impl="simt", images=(4, 20), T=2, ties="zero"),
    "b1": dict(mode="beam", prec="bf16", impl="tc", images=(6, 44), rpi=1, T=4),
    "b3_div_u": dict(mode="beam", prec="fp32", impl="simt", images=(4, 44), rpi=3, T=4, div="u"),
    "b3_div_philox": dict(mode="beam", prec="bf16", impl="tc", images=(4, 44), rpi=3, T=4, div="philox"),
    "b5": dict(mode="beam", prec="bf16", impl="tc", images=(8, 44), rpi=5, T=5, end_bias=0.5),
    "b5_alpha": dict(mode="beam", prec="bf16", impl="simt", images=(6, 44), rpi=5, T=4, alpha=0.6, end_bias=1.0),
    "b5_beta": dict(mode="beam", prec="bf16", impl="tc", images=_RAGGED, rpi=5, T=4, beta=0.3, end_bias=0.5),
    "b5_pen_ragged": dict(mode="beam", prec="bf16", impl="tc", images=_RAGGED, rpi=5, T=5, alpha=0.6, beta=0.3, end_bias=1.0),
    "b16": dict(mode="beam", prec="fp32", impl="simt", images=(4, 30), rpi=16, T=3, alpha=0.6, beta=0.3),
    "b16_tc": dict(mode="beam", prec="bf16", impl="tc", images=(5, 30), rpi=16, T=3),
    "b5_dup": dict(mode="beam", prec="bf16", impl="tc", images=(4, 44), rpi=5, T=3, ties="dup"),
    "b4_zero": dict(mode="beam", prec="fp32", impl="simt", images=(3, 20), rpi=4, T=3, ties="zero", alpha=0.6),
    "b5_1025": dict(mode="beam", prec="bf16", impl="tc", images=(205, 16), rpi=5, T=3),
    "b5_bench": dict(mode="beam", prec="bf16", impl="tc", images=(51, 372), rpi=5, T=3),
    # the two-layer decoder of the extension (lo_decoder2_greedy / _beam / _sample): layer 1 as above, layer 2 and its slots
    "l2_g_ragged": dict(mode="greedy", prec="bf16", impl="tc", images=_RAGGED, T=4, end_bias=0.15, l2=True),
    "l2_b5_pen": dict(mode="beam", prec="bf16", impl="tc", images=(6, 44), rpi=5, T=4, alpha=0.6, beta=0.3, end_bias=0.2, l2=True),
    "l2_b3_fp32": dict(mode="beam", prec="fp32", impl="simt", images=_RAGGED, rpi=3, T=3, div="u", l2=True),
    "l2_s8": dict(mode="sample", prec="bf16", impl="simt", images=(4, 44), rpi=8, T=3, tau=1.0, k=0, p=0.9, u="philox", l2=True),
    "s1_k1": dict(mode="sample", prec="bf16", impl="tc", images=(8, 44), rpi=1, T=4, tau=1.0, k=1, p=1.0, u="u"),
    "s8_kV": dict(mode="sample", prec="bf16", impl="tc", images=(4, 44), rpi=8, T=4, tau=1.0, k=500, p=1.0, u="philox",
                  end_bias=2.0),
    "s8_k5": dict(mode="sample", prec="fp32", impl="simt", images=(4, 44), rpi=8, T=4, tau=1.0, k=5, p=1.0, u="u"),
    "s8_p_one": dict(mode="sample", prec="bf16", impl="tc", images=(4, 44), rpi=8, T=3, tau=1.0, k=0, p=1e-6, u="philox"),
    "s8_p_boundary": dict(mode="sample", prec="fp32", impl="simt", images=(3, 20), rpi=8, T=3, tau=1.0, k=0, p=0.25, u="u",
                          ties="zero"),
    "s8_p09_ragged": dict(mode="sample", prec="bf16", impl="tc", images=_RAGGED, rpi=8, T=4, tau=1.0, k=0, p=0.9, u="philox",
                          end_bias=2.0),
    "s8_p_exact": dict(mode="sample", prec="fp32", impl="simt", images=(3, 20), rpi=8, T=2, tau=1.0, k=0, p=0.25, u="u",
                       ties="const", u_peak=125),
    "s8_tau05": dict(mode="sample", prec="bf16", impl="simt", images=(4, 44), rpi=8, T=3, tau=0.5, k=0, p=1.0, u="u"),
    "s8_tau2": dict(mode="sample", prec="bf16", impl="tc", images=(4, 44), rpi=8, T=3, tau=2.0, k=20, p=0.8, u="philox"),
    "s8_V501": dict(mode="sample", prec="bf16", impl="tc", images=(3, 44), rpi=8, T=3, V=501, tau=1.0, k=0, p=0.95, u="philox"),
    "s8_V2048": dict(mode="sample", prec="bf16", impl="tc", images=(3, 44), rpi=8, T=3, V=2048, tau=1.0, k=0, p=0.9, u="philox"),
}

# schedule -> (library options, the cases it runs); the options a decode reads: the per-step GEMMs (skinny_*), PDL, and the
# attention forward (att_pipe, att_nsplit, att_cluster, att_l2_keep_mb, deterministic)
_SCHEDULES = {
    "default": ({}, list(_CASES)),
    "skinny_mma0": ({"skinny_mma": 0}, ["g_tc72", "b5", "s8_tau2"]),
    "skinny_tma0": ({"skinny_tma": 0}, ["g_tc72", "b5_pen_ragged"]),
    "skinny8_0": ({"skinny8": 0}, ["g_tc72", "b5"]),
    "pdl0": ({"pdl": 0}, ["g_tc_ragged", "b5_pen_ragged", "s8_p09_ragged", "l2_b5_pen"]),
    "att_pipe0": ({"att_pipe": 0}, ["g_tc72", "b5", "s8_tau2"]),
    "att_nsplit1": ({"att_nsplit": 1}, ["g_tc_ragged", "b5_pen_ragged"]),
    "att_nsplit3": ({"att_nsplit": 3}, ["g_tc72", "b5_pen_ragged"]),
    "att_cluster0": ({"att_cluster": 0}, ["b5", "g_tc72"]),
    "att_l2_keep0": ({"att_l2_keep_mb": 0}, ["b5_bench"]),
    "deterministic": ({"deterministic": 1}, ["g_tc_ragged", "b5_pen_ragged", "b3_div_philox", "s8_p09_ragged", "l2_b5_pen"]),
}
_PARAMS = [(s, c) for s, (_, cs) in _SCHEDULES.items() for c in cs]

_WORST = {}
_INSIDE = {}
_SEED = 0x5EED1234


def _model(case, seed):
    from latex_ocr_b200.decoder import DecoderWithAttention
    cfg = _CASES[case]
    V = cfg.get("V", 500)
    torch.manual_seed(seed)
    dec = DecoderWithAttention(512, _E, 512, V, encoder_dim=512, dropout=0.5, device="cuda", precision=cfg["prec"],
                               impl=cfg["impl"])
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    with torch.no_grad():
        fw, fb = dec.fc.weight, dec.fc.bias
        fw.uniform_(-0.15, 0.15, generator=g)
        fb.uniform_(-0.1, 0.1, generator=g)
        if "end_bias" in cfg:
            fb[END] = cfg["end_bias"]
        if cfg.get("ties") == "dup":
            fw[10:20] = fw[10].clone()
            fb[10:20] = 1.0
        elif cfg.get("ties") == "const":
            fw.zero_()
            fb.fill_(0.3)
        elif cfg.get("ties") == "zero":
            fw.zero_()
            fb.copy_((torch.randint(0, 4, (V,), device="cuda", generator=g) * 0.25).float())
            fb[END] = -1.0
        dec.store.refresh_shadow()
    images = cfg["images"]
    counts = [images[1]] * images[0] if isinstance(images, tuple) else list(images)
    enc = [torch.relu(torch.randn(n, 512, device="cuda", generator=g)).to(dec.tdtype) for n in counts]
    layer2 = None
    if cfg.get("l2"):
        from latex_ocr_b200.ext import DecoderLayer2
        layer2 = DecoderLayer2(512, device="cuda", precision=cfg["prec"], impl=cfg["impl"])
    return dec, enc, counts, layer2


def _l2_views(scratch, B, D):
    """layer 2's scratch (csrc/lo_decoder2.cuh dec2_carve): gates [B][4D], h and c [2][B][D], the bf16 mirror of h [2][B][D]"""
    al = lambda n: (n + 255) // 256 * 256
    n = B * D
    o_h = al(16 * n)
    o_c = o_h + al(8 * n)
    o_b = o_c + al(8 * n)
    f = lambda o, k: scratch[o:o + 4 * k].view(torch.float32)
    return dict(gates=f(0, 4 * n).view(B, 4 * D), h=f(o_h, 2 * n).view(2, B, D), c=f(o_c, 2 * n).view(2, B, D),
                h_bf=scratch[o_b:o_b + 4 * n].view(torch.bfloat16).view(2, B, D))


def _prepare(dec, enc, counts, rpi, T):
    """the workspace and args of a decode of the images ``enc`` (a list of [R_i][C]), through decode._prepare's own helpers"""
    from latex_ocr_b200 import decode
    N, R = len(enc), max(counts)
    off = decode.region_offsets(counts) if len(set(counts)) > 1 else None
    ws = decode.decode_workspace(dec, N, R, rpi, T, off)
    if off is not None:
        x = ws["t"]["enc"]
        x[:off[-1]].copy_(torch.cat(enc))
    else:
        x = ws["x"] = torch.stack(enc).contiguous()
    return decode.decode_args(dec, ws, x, N, R, rpi, T, off), ws


_STEP_BUFS = ("hall", "call", "out1", "alphas", "ctx", "gctx", "gates")


def _hall_mirror(ws, a):
    """the bf16 mirror of hall [T+1][B][D] inside bfwork (csrc/lo_decoder.cu bf_views)"""
    bf = ws["t"]["bfwork"].view(torch.bfloat16)
    o = a.T * a.B * (a.A + a.C + 4 * a.D)
    return bf[o:o + (a.T + 1) * a.B * a.D].view(a.T + 1, a.B, a.D)


def _run(case, dec, a, ws, T, extra, layer2=None):
    """the decode call with max_steps = 1 .. T from sentinel-filled buffers; returns one snapshot per call"""
    from latex_ocr_b200 import _lib
    from latex_ocr_b200._lib import stream_ptr
    L = _lib.lib()
    cfg = _CASES[case]
    t_ = ws["t"]
    B, V, R = a.B, a.V, a.R
    tc = bool(a.impl == _lib.LO_IMPL_TC and a.dt == _lib.LO_BF16)
    snaps = []
    l2 = layer2.decode_layer(a) if layer2 is not None else None
    scratch = layer2._scratch.get(int(L.lo_decoder2_scratch_bytes(ctypes.byref(a)))) if layer2 is not None else None
    for n in range(1, T + 1):
        for k in _STEP_BUFS + ("logits", "row_loss", "mean", "sreg"):
            t_[k].fill_(SENTINEL)
        if tc:
            _hall_mirror(ws, a).fill_(SENTINEL)
        if scratch is not None:
            v = _l2_views(scratch, B, a.D)
            for k in ("gates", "h", "c"):
                v[k].fill_(SENTINEL)
            v["h_bf"].fill_(SENTINEL)
        s = {}
        if cfg["mode"] == "greedy":
            tokens = torch.full((B, n), -7, dtype=torch.int64, device="cuda")
            fin = torch.full((B,), 5, dtype=torch.int32, device="cuda")          # the call zeroes it
            hist = torch.full((B, n), -7, dtype=torch.int32, device="cuda")
            if l2 is not None:
                rc = L.lo_decoder2_greedy(ctypes.byref(a), ctypes.byref(l2), START, END, n, tokens.data_ptr(), fin.data_ptr(),
                                          hist.data_ptr(), stream_ptr())
            else:
                rc = L.lo_decoder_greedy_hist(ctypes.byref(a), START, END, n, tokens.data_ptr(), fin.data_ptr(), hist.data_ptr(),
                                              stream_ptr())
            s.update(tokens=tokens, fin_hist=hist, finished=fin)
        elif cfg["mode"] == "sample":
            sa = _lib.SampleArgs()
            sa.tau, sa.top_k, sa.top_p = cfg["tau"], cfg["k"], cfg["p"]
            logp = torch.full((B,), 17.0, device="cuda")                        # the call zeroes it
            sa.logp = logp.data_ptr()
            if cfg["u"] == "u":
                sa.u = extra["u"].data_ptr()
            else:
                extra["state"].copy_(extra["state0"])
                sa.state = extra["state"].data_ptr()
            tokens = torch.full((B, n), -7, dtype=torch.int64, device="cuda")
            fin = torch.full((B,), 5, dtype=torch.int32, device="cuda")
            hist = torch.full((B, n), -7, dtype=torch.int32, device="cuda")
            if l2 is not None:
                rc = L.lo_decoder2_sample(ctypes.byref(a), ctypes.byref(l2), ctypes.byref(sa), START, END, n, tokens.data_ptr(),
                                          fin.data_ptr(), hist.data_ptr(), stream_ptr())
            else:
                rc = L.lo_decoder_sample(ctypes.byref(a), ctypes.byref(sa), START, END, n, tokens.data_ptr(), fin.data_ptr(),
                                         hist.data_ptr(), stream_ptr())
            s.update(tokens=tokens, fin_hist=hist, finished=fin, logp=logp)
            if cfg["u"] != "u":
                s["state_after"] = extra["state"].clone()
        else:
            beam = a.rows_per_img
            N = B // beam
            ids = torch.full((N, n, beam), -7, dtype=torch.int64, device="cuda")
            parents = torch.full_like(ids, -7)
            hist = torch.full((N, n, beam), -7, dtype=torch.int32, device="cuda")
            logp = torch.full((B,), 17.0, device="cuda")
            pt = extra["pen_t"]
            for k in pt:
                if k != "len_pen":
                    pt[k].fill_(-5 if pt[k].dtype == torch.int32 else SENTINEL)
            u = extra.get("div_u")
            st = None
            if cfg.get("div") == "philox":
                extra["state"].copy_(extra["state0"])
                st = extra["state"].data_ptr()
            gamma, prob = extra["div"]
            args = (START, END, n, ids.data_ptr(), parents.data_ptr(), hist.data_ptr(), logp.data_ptr(), gamma, prob,
                    u.data_ptr() if u is not None else None, st, ctypes.byref(extra["pen"]), stream_ptr())
            if l2 is not None:
                rc = L.lo_decoder2_beam(ctypes.byref(a), ctypes.byref(l2), *args)
            else:
                rc = L.lo_decoder_beam_pen(ctypes.byref(a), *args)
            rl = t_["row_loss"].view(torch.int32)
            s.update(ids=ids, parents=parents, fin_hist=hist, logp=logp, finished=rl[:B].clone(), parent_rows=rl[B:2 * B].clone(),
                     pen={k: v.clone() for k, v in pt.items()})
        assert rc == 0, L.lo_last_error()
        torch.cuda.synchronize()
        s["logits"] = t_["logits"].view(-1)[:B * V].view(B, V).clone()
        s["next_tok"] = t_["sreg"].view(-1)[:2 * B].view(torch.int64).clone()
        for k in _STEP_BUFS + ("mean",):
            s[k] = t_[k].clone()
        if tc:
            s["hall_bf"] = _hall_mirror(ws, a).clone()
        if scratch is not None:
            s["l2"] = {k: v.clone() for k, v in _l2_views(scratch, B, a.D).items()}
        snaps.append(s)
    return snaps


def _outputs_of(s):
    return [s[k] for k in ("tokens", "ids", "parents", "fin_hist") if k in s] + [s[k] for k in _STEP_BUFS]


def _check_prefix(case, snaps):
    """every shorter call's outputs and per-step buffers are a bit-for-bit prefix of the longest call's"""
    F = snaps[-1]
    T = len(snaps)
    for n, s in enumerate(snaps, 1):
        for k in ("tokens", "fin_hist"):
            if k in s and s[k].dim() == 2:
                assert torch.equal(s[k], F[k][:, :n]), "%s: %s of max_steps=%d is not a prefix" % (case, k, n)
        for k in ("ids", "parents", "fin_hist"):
            if k in s and s[k].dim() == 3:
                assert torch.equal(s[k], F[k][:, :n]), "%s: %s of max_steps=%d is not a prefix" % (case, k, n)
        for k, sl in (("hall", slice(0, n + 1)), ("call", slice(0, n + 1)), ("out1", slice(0, n)), ("ctx", slice(0, n)),
                      ("gctx", slice(0, n)), ("gates", slice(0, n))):
            assert torch.equal(bits(s[k][sl]), bits(F[k][sl])), "%s: %s of max_steps=%d is not a prefix" % (case, k, n)
        assert torch.equal(bits(s["alphas"][:, :n]), bits(F["alphas"][:, :n])), "%s: alphas prefix (%d)" % (case, n)
        if n < T:
            for k in ("out1", "ctx", "gctx", "gates"):
                assert bool((s[k][n:] == SENTINEL).all()), "%s: %s past max_steps=%d written" % (case, k, n)


def _signature(x):
    """[M] int64: equal for the rows of x [M][..] that are equal (candidates computed from the same fp32 inputs)"""
    return torch.unique(x.reshape(x.shape[0], -1), dim=0, return_inverse=True)[1]


def _kept(x, tau, top_k, top_p):
    """(surely kept, possibly kept) [V] bool: the filter of one row under fp32.  The top-k part is exact (a sort of the fp32
    logits); the top-p cut falls where the mass before a position reaches top_p, and that mass errs by at most (V + 10) 2^-23 of
    itself (sums of expf, over sq).  Both contain tests/sample_oracle.keep_mask's set.  A row of equal logits is exact in fp32
    (every expf is 1, the masses are i / V with one rounding): there the cut is the first position i with fl32(i / V) >= top_p."""
    import sample_oracle as so
    V = len(x)
    if (x == x[0]).all():
        pos = np.float32(np.arange(V)) / np.float32(V) < np.float32(top_p)
        if top_k > 0:
            pos &= np.arange(V) < top_k
        return pos.copy(), pos.copy()
    z = x / tau
    q = np.exp(z - z.max())
    q /= q.sum()
    order = np.lexsort((np.arange(V), -q))
    before = np.concatenate(([0.0], np.cumsum(q[order])[:-1]))
    pos = np.ones(V, dtype=bool)
    if top_k > 0:
        pos &= np.arange(V) < top_k
    lo_pos, hi_pos = pos.copy(), pos.copy()
    if top_p < 1.0:
        tol = before * (V + 10) * 2.0 ** -23 + 2.0 ** -40
        lo_pos &= before + tol < top_p
        hi_pos &= before - tol < top_p
    lo, hi = np.zeros(V, dtype=bool), np.zeros(V, dtype=bool)
    lo[order[lo_pos]] = True
    hi[order[hi_pos]] = True
    mid, _ = so.keep_mask(x, tau, top_k, top_p)
    assert not (lo & ~mid).any() and not (mid & ~hi).any()
    return lo, hi


def _decide(ck, name, K, E, chosen, sig):
    """the top-k decision rule on one image: K, E [M] float64 keys and fp32 allowances, chosen [k] the kernel's flat indices in
    its order, sig [M] equal for candidates computed from the same fp32 inputs (whose keys tie bit for bit in the kernel too).
    Returns the number of decisions taken inside the margin."""
    taken = torch.zeros_like(K, dtype=torch.bool)
    inside = 0
    idx = torch.arange(K.numel(), device=K.device)
    for i in chosen.tolist():
        assert 0 <= i < K.numel() and not bool(taken[i]), "%s %s: chosen index %d repeated or out of range" % (ck.tag, name, i)
        rest = ~taken
        rest[i] = False
        better = rest & (K - E > K[i] + E[i])
        assert not bool(better.any()), "%s %s: picked %d (key %r +- %.3g) over %d (key %r +- %.3g)" % (
            ck.tag, name, i, K[i].item(), E[i].item(), int(better.nonzero()[0]), K[better][0].item(), E[better][0].item())
        tie_lower = rest & (sig == sig[i]) & (idx < i)
        assert not bool(tie_lower.any()), "%s %s: tie at key %r went to %d before the lower index %d" % (
            ck.tag, name, K[i].item(), i, int(tie_lower.nonzero()[0]))
        close = rest & (K + E >= K[i] - E[i]) & (K != K[i])
        inside += int(bool(close.any()))
        taken[i] = True
    return inside


def _lsm_allowance(lse, lp, V):
    return (V + 8) * 2.0 ** -24 + 2.0 ** -23 * lse.abs() + 2.0 ** -24 * lp.abs()


def _choose(ck, cfg, t, s, prev, lg, fin_prev, logp_prev, al_k, counts, extra):
    """the choice of step t on the kernel's own logits lg [B][V] (see the module docstring); s / prev: the snapshots of the
    calls of t + 1 and t steps (prev None at t = 0).  Returns (finished after step t, logp after step t, decisions inside the
    margin)."""
    mode = cfg["mode"]
    B, V = lg.shape
    R = al_k.shape[1]
    beam = s["ids"].shape[2] if mode == "beam" else 1
    N = B // beam
    Ri = torch.tensor(counts, device="cuda").repeat_interleave(B // len(counts))
    lgd = lg.double()
    inside = 0
    if mode == "greedy":
        want = dr.greedy(lg.cpu().double(), fin_prev.cpu(), END)[0].cuda()     # the first maximum
        got = s["tokens"][:, t]
        assert torch.equal(got, want), "%s: greedy argmax differs at step %d rows %s" % (
            ck.tag, t, (got != want).nonzero()[:, 0].tolist()[:8])
        fin_now = fin_prev | (want == END)
        assert torch.equal(s["fin_hist"][:, t].bool(), fin_now), "%s: finished flags at step %d" % (ck.tag, t)
        assert torch.equal(s["next_tok"], want)
    elif mode == "sample":
        tau, k_, p_ = cfg["tau"], cfg["k"], cfg["p"]
        u = extra["u"][t].double() if cfg["u"] == "u" else dr.philox_uniforms(_SEED, 3, t, B, V).cuda()
        got = s["tokens"][:, t]
        lse = torch.logsumexp(lgd, -1)
        gs = -torch.log(-torch.log(u))
        sc = lgd / tau + gs
        e_sc = 2.0 ** -22 * ((lgd / tau).abs() + gs.abs() + 1)
        x = lgd.cpu().numpy()
        for b in range(B):
            if bool(fin_prev[b]):
                assert int(got[b]) == END, "%s: a finished row sampled %d" % (ck.tag, int(got[b]))
                continue
            lo, hi = _kept(x[b], tau, k_, p_)
            inside += int(not np.array_equal(lo, hi))      # a top-p cut within the fp32 margin: either side is accepted
            hi_t, lo_t = torch.from_numpy(hi).cuda(), torch.from_numpy(lo).cuda()
            assert bool(hi_t[got[b]]), "%s: row %d step %d sampled %d outside the kept set" % (ck.tag, b, t, int(got[b]))
            lo_t[got[b]] = True
            K = torch.where(lo_t, sc[b], torch.full_like(sc[b], -math.inf))
            Eb = torch.where(lo_t, e_sc[b], torch.zeros_like(sc[b]))
            sig = _signature(torch.stack([lgd[b], u[b]], 1))
            inside += _decide(ck, "sample draw", K, Eb, got[b:b + 1], sig)
        fin_now = fin_prev | (got == END)
        assert torch.equal(s["fin_hist"][:, t].bool(), fin_now)
        assert torch.equal(s["next_tok"], got)
        lp_tok = lgd.gather(1, got[:, None])[:, 0] - lse
        live = ~fin_prev
        want_lp = torch.where(live, logp_prev + lp_tok, logp_prev)
        e_lp = torch.where(live, _lsm_allowance(lse, lp_tok, V) + 2.0 ** -24 * want_lp.abs(), torch.zeros_like(lse))
        ck.bound("sample logp", s["logp"], want_lp, e_lp)
        ck.exact("logp of finished rows", s["logp"][fin_prev], prev["logp"][fin_prev] if prev else torch.zeros(0, device="cuda"))
        logp_prev = s["logp"].double()
        fin_prev = fin_now
    else:
        pt = s["pen"]
        alpha_w, beta_w = cfg.get("alpha", 0.0), cfg.get("beta", 0.0)
        pen_on = alpha_w != 0 or beta_w > 0
        gamma, prob = extra["div"]
        div_on = not (gamma == 1 or prob == 0)
        lg_gamma = float(np.float32(math.log(gamma))) if div_on else 0.0
        u = None
        if div_on:
            u = extra["div_u"][t].double() if cfg["div"] == "u" else dr.div_philox_uniforms(_SEED, 3, t, B, V).cuda()
        len_in = None
        term = None
        nc = B * R
        if pen_on:
            h = t & 1
            len_in = prev["pen"]["len"][(1 - h) * B:(2 - h) * B] if t else torch.zeros(B, dtype=torch.int32, device="cuda")
            if beta_w > 0:
                cov_out = pt["cov"][h * nc:(h + 1) * nc].view(B, R)
                term = pt["cov"][2 * nc:2 * nc + B]
                cov_in = prev["pen"]["cov"][(1 - h) * nc:(2 - h) * nc].view(B, R) if t else None
                cref, _, _ = dr.coverage(al_k, cov_in, prev["parent_rows"] if t else None, fin_prev, counts, beam, t, beta_w)
                okm = torch.arange(R, device="cuda")[None, :] < Ri[:, None]
                ck.bound("coverage", cov_out[okm], cref[okm], 2.0 ** -24 * cref[okm].abs() + 1e-38)
                lnc = torch.where(okm, torch.log(cov_out.double().clamp(1e-30, 1.0)), torch.zeros_like(cref))
                tref = beta_w * lnc.sum(1)
                ck.bound("coverage term", term, tref, (ACC + 2.0 ** -22) * beta_w * lnc.abs().sum(1) + 2.0 ** -24 * tref.abs()
                         + 1e-38)
        LP = extra["pen_t"]["len_pen"].double() if alpha_w != 0 else None
        o = dr.beam_step(lgd, logp_prev, fin_prev, t, beam, END, lg_gamma, prob if div_on else 0.0, u, LP, term,
                         len_in if pen_on else None)
        # allowances of every candidate's total and key
        E_tot = _lsm_allowance(o["lse"], o["lp"], V) + 2.0 ** -24 * o["total"].abs()
        masked = o["lp"] <= -dr.FLT_MAX
        if div_on:
            # the rank is uncertain by the other candidates of the row whose pre-penalty totals lie within the allowances
            nb = o["nb"]
            pre_t = (logp_prev[:, None] + dr.log_softmax(lgd)[0]).view(N, beam, V)[:, :nb]
            e_pre = _lsm_allowance(dr.log_softmax(lgd)[1][:, None], dr.log_softmax(lgd)[0], V).view(N, beam, V)[:, :nb]
            d = (pre_t[..., :, None] - pre_t[..., None, :]).abs()
            unc = ((d <= e_pre[..., :, None] + e_pre[..., None, :]) & (d > 0)).sum(-1).double().reshape(N, nb * V)
            unc = unc * (prob > u).double().view(N, beam, V)[:, :nb].reshape(N, nb * V)      # only where the penalty applies
            E_tot = E_tot + abs(lg_gamma) * unc + 2.0 ** -23 * o["total"].abs()
        E_key = E_tot
        if pen_on:
            if LP is not None:
                E_key = E_key / float(LP.min()) + 2.0 ** -24 * o["key"].abs()
            if term is not None:
                E_key = E_key + 2.0 ** -24 * o["key"].abs()
        E_key = torch.where(masked, torch.zeros_like(E_key), E_key)
        E_tot = torch.where(masked, torch.zeros_like(E_tot), E_tot)
        ids_k = s["ids"][:, t]
        par_k = s["parents"][:, t]
        flat = par_k * V + ids_k
        # candidates computed from the same fp32 inputs: the logits row (as a class of equal rows), the token's logit,
        # logp, finished, len_in, the coverage term and the diversity penalty applied
        nb = o["nb"]
        cls = _signature(lgd)[:, None].expand(B, V)
        cols = [cls, lgd, logp_prev[:, None].expand(B, V), fin_prev.double()[:, None].expand(B, V)]
        if len_in is not None:
            cols.append(len_in.double()[:, None].expand(B, V))
        if term is not None:
            cols.append(term.double()[:, None].expand(B, V))
        if div_on:
            rank = dr.div_ranks((logp_prev[:, None] + dr.log_softmax(lgd)[0]).view(N, beam, V)).view(B, V)
            cols.append(torch.where(prob > u, rank, torch.full_like(lgd, -1.0)))
        sigs = torch.stack([c.reshape(N, beam, V)[:, :nb].reshape(N, nb * V) for c in cols], -1)
        for i in range(N):
            inside += _decide(ck, "beam top-k", o["key"][i], E_key[i], flat[i], _signature(sigs[i]))
        ar = torch.arange(N, device="cuda")[:, None]
        rows = (par_k + ar * beam).reshape(-1)
        fin_par = fin_prev[rows].view(N, beam)
        fin_now = (fin_par | (ids_k == END)).reshape(-1)
        assert torch.equal(s["fin_hist"][:, t].reshape(-1).bool(), fin_now), "%s: fin_hist at step %d" % (ck.tag, t)
        assert torch.equal(s["finished"].bool(), fin_now)
        assert torch.equal(s["next_tok"], ids_k.reshape(-1))
        assert torch.equal(s["parent_rows"].long(), rows), "%s: parent_rows at step %d" % (ck.tag, t)
        if pen_on:
            lin = len_in.long()[rows].view(N, beam)
            want_len = (lin + (~fin_par & (ids_k != END)).long()).reshape(-1)
            assert torch.equal(pt["len"][(t & 1) * B:((t & 1) + 1) * B].long(), want_len), "%s: len_out at step %d" % (ck.tag, t)
        tot_c = o["total"].gather(1, flat).reshape(-1)
        key_c = o["key"].gather(1, flat).reshape(-1)
        ck.bound("beam logp", s["logp"], tot_c, E_tot.gather(1, flat).reshape(-1) + 1e-30)
        if "scores" in pt:
            ck.bound("beam scores", pt["scores"].reshape(-1), key_c, E_key.gather(1, flat).reshape(-1) + 1e-30)
        logp_prev = s["logp"].double()
        fin_prev = fin_now
    if mode == "greedy":
        logp_prev = None
    return fin_now, logp_prev, inside


def _check_layer2(ck, layer2, s, prev, F, t, pr, mode, act, tc, p):
    """layer 2 of step t (two-layer decoder) from the snapshots s / prev of the calls of t + 1 and t steps: the slot it read (the
    zero state at t = 0), its gates from h1 and that h2, c2 and h2 from its own gates, the bf16 mirror, the logits fc(h2) of every
    row; in beam search h1 before the gather survives for the parent rows only (their gates are checked), step t writes slot 1
    and the reorder gathers it into slot 0 by parent_rows, bit for bit with the mirror recast"""
    S2 = layer2.store
    w_ih, w_hh = S2.w("cell.weight_ih").double(), S2.w("cell.weight_hh").double()
    bsum = S2.f32("cell.bias_ih").double() + S2.f32("cell.bias_hh").double()
    v = s["l2"]
    if mode == "beam":
        cur, rd = 1, 0
        h_rd = prev["l2"]["h"][rd] if t else torch.zeros_like(v["h"][0])
        c_rd = prev["l2"]["c"][rd] if t else torch.zeros_like(v["c"][0])
    else:
        cur, rd = (t + 1) & 1, t & 1
        h_rd = v["h"][rd] if t else torch.zeros_like(v["h"][0])
        c_rd = v["c"][rd] if t else torch.zeros_like(v["c"][0])
    # layer 1's h of step t before any gather: row q = the gathered row of a slot whose parent is q
    first = {}
    for b, q in enumerate(pr.tolist()):
        first.setdefault(q, b)
    rows = torch.tensor(sorted(first), device="cuda")
    src = torch.tensor([first[q] for q in sorted(first)], device="cuda")
    x1, S1 = ds.linear(act(F["hall"][t + 1][src]), w_ih)
    x2, S2_ = ds.linear(act(h_rd[rows]), w_hh)
    check_gates(ck, v["gates"][rows], x1 + x2 + bsum, ACC * (S1 + S2_ + bsum.abs()))
    i, f, g, o = v["gates"].double().chunk(4, 1)
    check_cell(ck, v["c"][cur], v["h"][cur], i, f, g, o, c_rd.double())
    if tc:
        ck.exact("bf16 mirror of h2", v["h_bf"][cur], v["h"][cur])
    ref, Sl = ds.linear(act(v["h"][cur]), p["fc.weight"], p["fc.bias"])
    ck.gemm("logits", s["logits"], ref, Sl)
    if mode == "beam":
        ck.exact("h2 gathered by parent", v["h"][0], v["h"][1][pr])
        ck.exact("c2 gathered by parent", v["c"][0], v["c"][1][pr])
        if tc:
            ck.exact("bf16 mirror of the gathered h2", v["h_bf"][0], v["h"][0])


def _check(ck, case, dec, a, ws, enc, counts, snaps, extra, layer2=None):
    from latex_ocr_b200 import _lib
    cfg = _CASES[case]
    S = dec.store
    F = snaps[-1]
    T = len(snaps)
    B, V, R, C, D, A = a.B, a.V, a.R, a.C, a.D, a.A
    rpi = max(1, a.rows_per_img)
    N = B // rpi
    tc = bool(a.impl == _lib.LO_IMPL_TC and a.dt == _lib.LO_BF16)
    act = rn if tc else (lambda x: x.double())
    names_w = ("attention.encoder_att.weight", "attention.decoder_att.weight", "f_beta.weight", "decode_step.weight_hh",
               "embedding.weight", "decode_step.weight_ih", "init_h.weight", "init_c.weight", "fc.weight")
    p = {n: S.w(n).double() for n in names_w}
    for n in ("attention.encoder_att.bias", "attention.decoder_att.bias", "f_beta.bias", "decode_step.bias_hh", "decode_step.bias_ih",
              "init_h.bias", "init_c.bias", "fc.bias", "attention.full_att.weight"):
        p[n] = S.f32(n).double()
    wf = p["attention.full_att.weight"].reshape(-1)
    wc, bc = ds.wcat(p)
    w_ctx = p["decode_step.weight_ih"][:, _E:]
    encd = [e.double() for e in enc]
    img = torch.arange(B, device="cuda") // rpi
    Ri = torch.tensor(counts, device="cuda")[img]

    # ---- prologue: the row means over each image's own regions, h0 and c0
    mean_ref = torch.stack([e.mean(0) for e in encd])[img]
    mean_S = torch.stack([e.abs().mean(0) for e in encd])[img]
    ck.bound("mean", F["mean"][:B], mean_ref, (Ri[:, None] + 1) * 2.0 ** -24 * mean_S)
    mean = F["mean"][:B].double()
    split = 2.0 ** -18 if (tc and C % 64 == 0 and a.T >= 2) else 0.0
    for k, nm in ((F["hall"][0], "init_h"), (F["call"][0], "init_c")):
        ref, Si = ds.linear(mean, p[nm + ".weight"], p[nm + ".bias"])
        ck.bound("h0 c0", k, ref, (ACC + split) * Si)
    ptab = ws["t"]["ptab"].double()
    att1 = ws["t"]["att1"]
    off = np.concatenate([[0], np.cumsum(counts)]).tolist()
    att1_img = [att1.view(-1)[off[i] * A:off[i + 1] * A].view(counts[i], A).double() for i in range(N)]
    ref, Sa = ds.linear(torch.cat(encd), p["attention.encoder_att.weight"], p["attention.encoder_att.bias"])
    from step_check import half_ulp_bf16
    ck.bound("att1", torch.cat([x for x in att1_img]), ref, ACC * Sa + (half_ulp_bf16(ref) if att1.dtype == torch.bfloat16 else 0))

    mode = cfg["mode"]
    fin_prev = torch.zeros(B, dtype=torch.bool, device="cuda")
    logp_prev = torch.zeros(B, dtype=torch.float64, device="cuda")
    inside = 0
    n_fin = []
    for t in range(T):
        s = snaps[t]
        prev = snaps[t - 1] if t else None
        # ---- the step: out1, attention per image, gates, cell
        h_prev = F["hall"][t]
        out1 = F["out1"][t]
        ref, S1 = ds.linear(act(h_prev), wc, bc)
        ck.gemm("out1 att2", out1[:, :A], ref[:, :A], S1[:, :A])
        ck.gemm("out1 hh", out1[:, A + C:], ref[:, A + C:], S1[:, A + C:])
        ck.bound("out1 gate", out1[:, A:A + C], torch.sigmoid(ref[:, A:A + C]), 0.25 * ACC * S1[:, A:A + C] + ULPS)
        att2, gate, hh = out1[:, :A].double(), out1[:, A:A + C].double(), out1[:, A + C:].double()
        al_k = F["alphas"][:, t]
        for i in range(N):
            r = slice(i * rpi, (i + 1) * rpi)
            n = counts[i]
            _, alpha, ctx, _ = ds.attention(att1_img[i].expand(rpi, -1, -1), encd[i].expand(rpi, -1, -1), att2[r], wf, gate[r])
            ck.attn("alphas", al_k[r, :n], alpha)
            ck.attn("ctx", F["ctx"][t][r], ctx)
            ck.attn("gctx", F["gctx"][t][r], gate[r] * F["ctx"][t][r].double())
            if n < R:
                ck.value("alphas past the image's regions", al_k[r, n:], SENTINEL)
        if t == 0:
            tok = torch.full((B,), START, dtype=torch.int64, device="cuda")
        else:
            tok = prev["next_tok"]
        pre_g, Sg = ds.linear(act(F["gctx"][t]), w_ctx)
        pre = pre_g + ptab[tok] + hh
        e_pre = ACC * (Sg + ptab[tok].abs() + hh.abs())
        gts = F["gates"][t]
        check_gates(ck, gts, pre, e_pre)
        i_, f_, g_, o_ = gts.double().chunk(4, 1)
        pr = s["parent_rows"].long() if mode == "beam" else torch.arange(B, device="cuda")
        check_cell(ck, F["call"][t + 1], F["hall"][t + 1], i_[pr], f_[pr], g_[pr], o_[pr], F["call"][t].double()[pr])
        if tc:
            ck.exact("bf16 mirror of hall", F["hall_bf"][t + 1], F["hall"][t + 1])
        # ---- beam search: the slots of one parent hold bit-identical state
        first = {}                                  # parent row -> its first slot
        for b, q in enumerate(pr.tolist()):
            first.setdefault(q, b)
        par = torch.tensor(sorted(first), device="cuda")
        src = torch.tensor([first[q] for q in sorted(first)], device="cuda")
        if mode == "beam":
            same = torch.tensor([first[q] for q in pr.tolist()], device="cuda")
            for k in ("hall", "call"):
                assert torch.equal(bits(F[k][t + 1]), bits(F[k][t + 1][same])), "%s: slots of one parent differ in %s" % (ck.tag, k)
        # ---- logits of step t from the kernel's own h (h2 in the two-layer decoder); in beam search the parent rows' h
        lg = s["logits"]
        if layer2 is not None:
            _check_layer2(ck, layer2, s, prev, F, t, pr, mode, act, tc, p)
        else:
            ref, Sl = ds.linear(act(F["hall"][t + 1]), p["fc.weight"], p["fc.bias"])
            ck.gemm("logits", lg[par], ref[src], Sl[src])

        # ---- the choice
        fin_now, logp_prev, ins = _choose(ck, cfg, t, s, prev, lg, fin_prev, logp_prev, al_k, counts, extra)
        inside += ins
        fin_prev = fin_now
        n_fin.append(int(fin_now.sum()))
    return inside, n_fin


def _extra(case, a):
    from latex_ocr_b200 import decode
    cfg = _CASES[case]
    B, V, T = a.B, a.V, _CASES[case]["T"]
    g = torch.Generator(device="cuda").manual_seed(99)
    x = {"state0": torch.tensor([_SEED, 3], dtype=torch.int64, device="cuda")}
    x["state"] = x["state0"].clone()
    if cfg["mode"] == "sample" and cfg["u"] == "u":
        x["u"] = torch.rand(T, B, V, device="cuda", generator=g).clamp_(1e-7, 1 - 2.0 ** -22)
        if "u_peak" in cfg:
            x["u"][:, :, cfg["u_peak"]] = 1 - 2.0 ** -24          # the token right past the top-p cut scores highest
    if cfg["mode"] == "beam":
        x["pen"], x["pen_t"] = decode.beam_penalty(cfg.get("alpha", 0.0), cfg.get("beta", 0.0), B, a.R, T, a.rows_per_img, "cuda")
        x["div"] = (0.5, 0.6) if "div" in cfg else (1.0, 0.0)
        if cfg.get("div") == "u":
            x["div_u"] = torch.rand(T, B, V, device="cuda", generator=g)
    return x


@pytest.mark.parametrize("schedule,case", _PARAMS, ids=["%s-%s" % sc for sc in _PARAMS])
def test_decode_steps_vs_float64(schedule, case):
    """Every decode step's state, logits and choice within the bounds of the module docstring of float64 from the kernel's own
    operands; shorter calls are bit-for-bit prefixes of longer ones.  Under "deterministic" two runs agree bit for bit."""
    from latex_ocr_b200 import _lib
    opts, _ = _SCHEDULES[schedule]
    cfg = _CASES[case]
    seed = sorted(_CASES).index(case)
    dec, enc, counts, layer2 = _model(case, seed)
    T = cfg["T"]
    with _lib.option(**opts):
        a, ws = _prepare(dec, enc, counts, cfg.get("rpi", 1), T)
        extra = _extra(case, a)
        snaps = _run(case, dec, a, ws, T, extra, layer2)
        _check_prefix(case, snaps)
        ck = Checker("%s %s" % (schedule, case))
        inside, n_fin = _check(ck, case, dec, a, ws, enc, counts, snaps, extra, layer2)
        if "deterministic" in opts:
            again = _run(case, dec, a, ws, T, extra, layer2)
            for x, y in zip(_outputs_of(snaps[-1]), _outputs_of(again[-1])):
                assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), "deterministic: two runs differ"
    for k, v in ck.worst.items():
        _WORST[k] = max(_WORST.get(k, 0.0), v)
    _INSIDE[case] = max(_INSIDE.get(case, 0), inside)
    print("\n%-34s finished per step %s, decisions inside the margin %d\n    %s" % (
        ck.tag, n_fin, inside, "  ".join("%s %.3f" % kv for kv in sorted(ck.worst.items()))))


# ---------------------------------------------------------------------------------------------------------------------------------
# the TensorFlow flavour (lo_tfdec_greedy, lo_tfdec_beam_pen, lo_tfdec_sample): every launch of every step from the workspace
# (tests/tfdec_step_ref.py carve), the reorder of xh, its mirror and c, and every choice on the kernel's own logits
# ---------------------------------------------------------------------------------------------------------------------------------
_TF_CASES = {
    "tf_g_ragged": dict(mode="greedy", prec="fp32", impl="simt", images=_RAGGED, rpi=1, T=4, end_bias=2.0),
    "tf_g_tc": dict(mode="greedy", prec="bf16", impl="tc", images=(8, 44), rpi=1, T=4),
    "tf_b5_pen": dict(mode="beam", prec="fp32", impl="simt", images=(4, 44), rpi=5, T=4, alpha=0.6, beta=0.3, end_bias=2.0),
    "tf_b5_tc": dict(mode="beam", prec="bf16", impl="tc", images=(6, 44), rpi=5, T=4, end_bias=2.0),
    "tf_b3_div_ragged": dict(mode="beam", prec="bf16", impl="tc", images=_RAGGED, rpi=3, T=3, div="philox"),
    "tf_b16": dict(mode="beam", prec="bf16", impl="tc", images=(3, 30), rpi=16, T=3, alpha=0.6),
    "tf_s8": dict(mode="sample", prec="bf16", impl="tc", images=(4, 44), rpi=8, T=3, tau=1.0, k=0, p=0.9, u="philox"),
    "tf_s8_ragged_fp32": dict(mode="sample", prec="fp32", impl="simt", images=_RAGGED, rpi=8, T=3, tau=0.5, k=20, p=1.0, u="u"),
}
_TF_SCHEDULES = {
    "default": ({}, list(_TF_CASES)),
    "skinny_mma0": ({"skinny_mma": 0}, ["tf_g_tc", "tf_s8"]),
    "pdl0": ({"pdl": 0}, ["tf_b3_div_ragged", "tf_b5_tc"]),
    "att_nsplit3": ({"att_nsplit": 3}, ["tf_b3_div_ragged", "tf_g_tc"]),
    "deterministic": ({"deterministic": 1}, ["tf_b3_div_ragged", "tf_b5_tc", "tf_s8"]),
}
_TF_PARAMS = [(s, c) for s, (_, cs) in _TF_SCHEDULES.items() for c in cs]
# the forward state of the workspace a decode writes: filled with the sentinel before every call
_TF_FILLED = ("att_img", "ptab", "xh", "call", "gates", "ztmp", "out2", "ctx", "oc", "mean", "initpre", "sinit", "xh_bf", "ctx_bf")
_TF_SNAP = ("att_img", "ptab", "xh", "call", "gates", "out2", "ctx", "mean", "initpre", "sinit", "xh_bf", "ctx_bf", "next_tok",
            "finished", "parent_rows")


def _tf_model(case, seed):
    from latex_ocr_b200.tf_decoder import Decoder
    from util import Cfg
    cfg = _TF_CASES[case]
    V = 500
    torch.manual_seed(seed)
    c = Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=10,
            decoding="beam_search" if cfg["mode"] == "beam" else "greedy", beam_size=cfg["rpi"])
    dec = Decoder(c, V, END, device="cuda", precision=cfg["prec"], impl=cfg["impl"])
    S = dec.store
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    with torch.no_grad():
        S.f32("lstm.bias").uniform_(-0.3, 0.3, generator=g)
        S.f32("y_W_o").mul_(4.0)                  # logits spread over a few units
        if "end_bias" in cfg:
            S.f32("y_W_o")[END] *= cfg["end_bias"]    # a wider END logit: some rows end early, at different steps
    dec.store.refresh_shadow()
    images = cfg["images"]
    counts = [images[1]] * images[0] if isinstance(images, tuple) else list(images)
    enc = [torch.relu(torch.randn(n, 512, device="cuda", generator=g)).to(dec.tdtype) for n in counts]
    return dec, enc, counts


def _tf_prepare(dec, enc, counts, rpi, T):
    from latex_ocr_b200 import decode
    N = len(enc)
    dec.store.refresh_shadow()
    if len(set(counts)) > 1:
        ws = dec.packed_workspace(counts, T, rpi)
        for i, e in enumerate(enc):
            ws["enc"][ws["off"][i]:ws["off"][i + 1]].copy_(e)
        L, ws, a = dec._args(ws["enc"], N * rpi, T, max(counts), rows_per_img=rpi, ws=ws)
        decode.set_region_offsets(a, ws["reg_off_host"], ws["reg_off"], ws["off"])
    else:
        x = torch.stack(enc).contiguous()
        L, ws, a = dec._args(x, N * rpi, T, counts[0], rows_per_img=rpi, decode=True)
        ws["enc"] = x
    return a, ws


def _tf_run(case, dec, a, ws, T, extra):
    """the TF entry point with max_steps = 1 .. T from sentinel-filled logits, alphas and forward state of the workspace; one
    snapshot per call of the outputs and of the workspace (through tests/tfdec_step_ref.py carve)"""
    from latex_ocr_b200 import _lib
    from latex_ocr_b200._lib import stream_ptr
    import tfdec_step_ref as ts
    L = _lib.lib()
    cfg = _TF_CASES[case]
    B, V = a.B, a.V
    layout, _ = ts.carve(B, a.T, a.R, a.C, a.A, a.D, a.O, a.E, V, a.ldl, a.dt == _lib.LO_BF16, a.rows_per_img)
    v = ts.views_of(ws["ws"], layout)
    snaps = []
    for n in range(1, T + 1):
        ws["logits"].fill_(SENTINEL)
        ws["alphas"].fill_(SENTINEL)
        for k in _TF_FILLED:
            if k in v:
                v[k].fill_(SENTINEL)
        for k in ("next_tok", "finished", "parent_rows"):
            v[k].fill_(-5)
        s = {}
        tokens = torch.full((B, n), -7, dtype=torch.int64, device="cuda")
        hist = torch.full((B, n), -7, dtype=torch.int32, device="cuda")
        if cfg["mode"] == "greedy":
            rc = L.lo_tfdec_greedy(ctypes.byref(a), END, n, tokens.data_ptr(), hist.data_ptr(), stream_ptr())
            s.update(tokens=tokens, fin_hist=hist)
        elif cfg["mode"] == "sample":
            sa = _lib.SampleArgs()
            sa.tau, sa.top_k, sa.top_p = cfg["tau"], cfg["k"], cfg["p"]
            logp = torch.full((B,), 17.0, device="cuda")
            sa.logp = logp.data_ptr()
            if cfg["u"] == "u":
                sa.u = extra["u"].data_ptr()
            else:
                extra["state"].copy_(extra["state0"])
                sa.state = extra["state"].data_ptr()
            rc = L.lo_tfdec_sample(ctypes.byref(a), ctypes.byref(sa), END, n, tokens.data_ptr(), hist.data_ptr(), stream_ptr())
            s.update(tokens=tokens, fin_hist=hist, logp=logp)
        else:
            beam = a.rows_per_img
            N = B // beam
            ids = torch.full((N, n, beam), -7, dtype=torch.int64, device="cuda")
            parents = torch.full_like(ids, -7)
            hist = torch.full((N, n, beam), -7, dtype=torch.int32, device="cuda")
            logp = torch.full((B,), 17.0, device="cuda")
            pt = extra["pen_t"]
            for k in pt:
                if k != "len_pen":
                    pt[k].fill_(-5 if pt[k].dtype == torch.int32 else SENTINEL)
            u = extra.get("div_u")
            st = None
            if cfg.get("div") == "philox":
                extra["state"].copy_(extra["state0"])
                st = extra["state"].data_ptr()
            gamma, prob = extra["div"]
            rc = L.lo_tfdec_beam_pen(ctypes.byref(a), END, n, ids.data_ptr(), parents.data_ptr(), hist.data_ptr(), logp.data_ptr(),
                                     gamma, prob, u.data_ptr() if u is not None else None, st, ctypes.byref(extra["pen"]),
                                     stream_ptr())
            s.update(ids=ids, parents=parents, fin_hist=hist, logp=logp, pen={k: x.clone() for k, x in pt.items()})
        assert rc == 0, L.lo_last_error()
        torch.cuda.synchronize()
        s.update({k: v[k].clone() for k in _TF_SNAP if k in v})
        s["logits"] = ws["logits"].view(-1)[:B * V].view(B, V).clone()
        s["alphas"] = ws["alphas"].view(-1)[:B * a.T * a.R].view(B, a.T, a.R).clone()
        snaps.append(s)
    return snaps


def _tf_check(ck, dec, a, enc, counts, snaps, mode):
    """every launch of the TF decode from the operands it read (the bounds of tests/test_gpu_tfdec_steps.py): the prologue (att_img
    per image, the token table, each row's own image mean, the initial state), and per step t the gates from xh[t] and the token
    the row was fed (row V, the start token, at t = 0), c and h from the kernel's own gates, out2, the attention over the row's own
    image (the tanh.approx rule), ctx and its mirror, o, and the logits.  Beam search: after the reorder xh[t+1] and call[t+1]
    are the cell of row parent_rows[b], slots of one parent are bit-identical, xh_bf[t+1] is RN_bf16(xh[t+1]) bit for bit, and
    the logits (and out2) of the parent rows are checked against the gathered state."""
    import tfdec_step_ref as ts
    from step_check import half_ulp_bf16
    S = dec.store
    F = snaps[-1]
    B, V, A, C, D, O, E, R = a.B, a.V, a.A, a.C, a.D, a.O, a.E, a.R
    rpi = max(1, a.rows_per_img)
    N = B // rpi
    tc = dec.impl == "tc" and dec.precision == "bf16"
    act = rn if tc else (lambda x: x.double())
    eps = 2.0 ** -10.98 if dec.precision == "bf16" else 2.0 ** -22
    p = {}
    for n in ("att_img.kernel", "att_h.kernel", "o_W_h", "lstm.kernel", "o_W_c", "y_W_o", "W_c_0", "W_h_0", "W_o_0"):
        p[n] = S.w(n).double().t()
    for n in ("embedding_table", "start_token"):
        p[n] = S.w(n).double()
    for n in ("att_beta", "lstm.bias", "b_c_0", "b_h_0", "b_o_0"):
        p[n] = S.f32(n).double()
    beta = p["att_beta"]
    KE = p["lstm.kernel"][E:]
    encd = [e.double() for e in enc]
    off = np.concatenate([[0], np.cumsum(counts)]).tolist()
    aflat = F["att_img"].reshape(-1)
    aimg = [aflat[off[i] * A:off[i + 1] * A].view(counts[i], A) for i in range(N)]
    img = torch.arange(B, device="cuda") // rpi
    Ri = torch.tensor(counts, device="cuda")[img]

    # ---- prologue
    ref, Sa = ts.linear(torch.cat(encd), p["att_img.kernel"])
    got = torch.cat(aimg)
    ck.bound("att_img", got, ref, ACC * Sa + (half_ulp_bf16(ref) if got.dtype == torch.bfloat16 else 0))
    emb = torch.cat([p["embedding_table"], p["start_token"][None]], 0)
    ref, Sp = ts.linear(emb, p["lstm.kernel"][:E], p["lstm.bias"])
    ck.gemm("ptab", F["ptab"], ref, Sp)
    mean_ref = torch.stack([e.mean(0) for e in encd])[img]
    mean_S = torch.stack([e.abs().mean(0) for e in encd])[img]
    ck.bound("mean", F["mean"], mean_ref, (Ri[:, None] + 1) * 2.0 ** -24 * mean_S)
    wi, bi = ts.w_init(p)
    ref, Si = ts.linear(F["mean"].double(), wi, bi)
    ck.gemm("initpre", F["initpre"], ref, Si)
    ck.bound("sinit", F["sinit"], torch.tanh(F["initpre"].double()), ULPS)
    s0 = F["sinit"]
    ck.exact("c0", F["call"][0], s0[:, :D])
    ck.exact("xh0 h", F["xh"][0][:, O:], s0[:, D:2 * D])
    ck.exact("xh0 o", F["xh"][0][:, :O], s0[:, 2 * D:])
    if tc:
        ck.exact("xh_bf 0", F["xh_bf"][0], F["xh"][0])

    ptab = F["ptab"].double()
    for t in range(len(snaps)):
        s = snaps[t]
        tok = torch.full((B,), V, dtype=torch.int64, device="cuda") if t == 0 else snaps[t - 1]["next_tok"]
        z, Sz = ts.linear(act(F["xh"][t]), KE)
        pt = ptab[tok]
        pre, e_pre = z + pt, ACC * (Sz + pt.abs())
        gts = F["gates"][t]
        for q, (fn, lip, sh) in enumerate(((torch.sigmoid, 0.25, 0.0), (torch.tanh, 1.0, 0.0), (torch.sigmoid, 0.25, 1.0),
                                           (torch.sigmoid, 0.25, 0.0))):
            sl = slice(q * D, (q + 1) * D)
            ck.bound("gates", gts[:, sl], fn(pre[:, sl] + sh), lip * e_pre[:, sl] + ULPS)
        pr = s["parent_rows"].long() if mode == "beam" else torch.arange(B, device="cuda")
        i, g, f, o = gts.double()[pr].chunk(4, 1)
        cp = F["call"][t].double()[pr]
        ck.bound("c", F["call"][t + 1], f * cp + i * g, 2.0 ** -22 * ((f * cp).abs() + (i * g).abs()) + 1e-38)
        href = o * torch.tanh(F["call"][t + 1].double())
        ck.bound("h", F["xh"][t + 1][:, O:], href, 2.0 ** -21 * href.abs() + 1e-38)
        # the rows whose state before the reorder survives: the parents, each read through its first slot
        first = {}
        for b, q in enumerate(pr.tolist()):
            first.setdefault(q, b)
        par = torch.tensor(sorted(first), device="cuda")
        src = torch.tensor([first[q] for q in sorted(first)], device="cuda")
        if mode == "beam":
            same = torch.tensor([first[q] for q in pr.tolist()], device="cuda")
            for k in ("xh", "call"):
                assert torch.equal(bits(F[k][t + 1]), bits(F[k][t + 1][same])), "%s: slots of one parent differ in %s" % (ck.tag, k)
        if tc:
            ck.exact("xh_bf", F["xh_bf"][t + 1], F["xh"][t + 1])
        ref, S2 = ts.linear(act(F["xh"][t + 1][src, O:]), ts.w_cat2(p))
        ck.gemm("out2", F["out2"][t][par], ref, S2)
        # attention of every row over its own image, from the kernel's own att_img and att_h
        att_h = F["out2"][t][:, :A].double()
        for n_ in range(N):
            r = slice(n_ * rpi, (n_ + 1) * rpi)
            pre_a = aimg[n_].double()[None] + att_h[r, None, :]
            post = torch.tanh(pre_a)
            d_r = ((eps * post.abs() + 2.0 ** -23 * pre_a.abs()) * beta.abs()).sum(-1) + ACC * (post * beta).abs().sum(-1)
            alpha = torch.softmax((post * beta).sum(-1), 1)
            e_al = alpha * (d_r + (alpha * d_r).sum(1, keepdim=True)) + ULPS * alpha
            ck.bound("alphas", s["alphas"][r, t, :counts[n_]], alpha, e_al + 1e-38)
            ctx = alpha @ encd[n_]
            e_ctx = e_al @ encd[n_].abs() + ACC * (alpha @ encd[n_].abs())
            ck.bound("ctx", F["ctx"][t][r], ctx, e_ctx + 1e-38)
        if tc:
            ck.exact("ctx_bf", F["ctx_bf"][t], F["ctx"][t])
        oc, Soc = ts.linear(act(F["ctx"][t]), p["o_W_c"])
        oref = torch.tanh(oc + F["out2"][t][:, A:].double())[pr]
        ck.bound("o", F["xh"][t + 1][:, :O], oref, (ACC * Soc[pr] + ULPS) + 2.0 ** -23 * oref.abs() + 1e-38)
        ref, Sl = ts.linear(act(F["xh"][t + 1][src, :O]), p["y_W_o"])
        ck.gemm("logits", s["logits"][par], ref, Sl)


def _tf_extra(case, a):
    from latex_ocr_b200 import decode
    cfg = _TF_CASES[case]
    B, V, T = a.B, a.V, cfg["T"]
    g = torch.Generator(device="cuda").manual_seed(98)
    x = {"state0": torch.tensor([_SEED, 3], dtype=torch.int64, device="cuda")}
    x["state"] = x["state0"].clone()
    if cfg["mode"] == "sample" and cfg["u"] == "u":
        x["u"] = torch.rand(T, B, V, device="cuda", generator=g).clamp_(1e-7, 1 - 1e-7)
    if cfg["mode"] == "beam":
        x["pen"], x["pen_t"] = decode.beam_penalty(cfg.get("alpha", 0.0), cfg.get("beta", 0.0), B, a.R, T, a.rows_per_img, "cuda")
        x["div"] = (0.5, 0.6) if "div" in cfg else (1.0, 0.0)
        if cfg.get("div") == "u":
            x["div_u"] = torch.rand(T, B, V, device="cuda", generator=g)
    return x


@pytest.mark.parametrize("schedule,case", _TF_PARAMS, ids=["%s-%s" % sc for sc in _TF_PARAMS])
def test_tf_decode_steps_vs_float64(schedule, case):
    """The TensorFlow flavour's greedy, beam and sampling decode: every launch of every step from the operands it read
    (_tf_check), every choice from the kernel's own logits by the rules of the module docstring, alphas past an image's regions
    untouched, shorter calls bit-for-bit prefixes of longer ones; under "deterministic" two runs agree bit for bit."""
    from latex_ocr_b200 import _lib
    opts, _ = _TF_SCHEDULES[schedule]
    cfg = _TF_CASES[case]
    dec, enc, counts = _tf_model(case, 100 + sorted(_TF_CASES).index(case))
    T = cfg["T"]
    with _lib.option(**opts):
        a, ws = _tf_prepare(dec, enc, counts, cfg["rpi"], T)
        extra = _tf_extra(case, a)
        snaps = _tf_run(case, dec, a, ws, T, extra)
        ck = Checker("%s %s" % (schedule, case))
        F = snaps[-1]
        for n, s in enumerate(snaps, 1):
            for k in ("tokens", "ids", "parents", "fin_hist"):
                if k in s:
                    assert torch.equal(s[k], F[k][:, :n]), "%s: %s of max_steps=%d is not a prefix" % (case, k, n)
            assert torch.equal(bits(s["alphas"][:, :n]), bits(F["alphas"][:, :n])), "%s: alphas prefix (%d)" % (case, n)
            for k, sl in (("xh", slice(0, n + 1)), ("call", slice(0, n + 1)), ("gates", slice(0, n)), ("out2", slice(0, n)),
                          ("ctx", slice(0, n))):
                assert torch.equal(bits(s[k][sl]), bits(F[k][sl])), "%s: %s of max_steps=%d is not a prefix" % (case, k, n)
        _tf_check(ck, dec, a, enc, counts, snaps, cfg["mode"])
        rpi = cfg["rpi"]
        fin = torch.zeros(a.B, dtype=torch.bool, device="cuda")
        logp = torch.zeros(a.B, dtype=torch.float64, device="cuda")
        inside = 0
        for t in range(T):
            al_k = F["alphas"][:, t]
            for i, n in enumerate(counts):
                if n < a.R:
                    ck.value("alphas past the image's regions", al_k[i * rpi:(i + 1) * rpi, n:], SENTINEL)
            fin, logp, ins = _choose(ck, cfg, t, snaps[t], snaps[t - 1] if t else None, snaps[t]["logits"], fin, logp, al_k, counts,
                                     extra)
            inside += ins
        if "deterministic" in opts:
            again = _tf_run(case, dec, a, ws, T, extra)
            for k in ("tokens", "ids", "parents", "fin_hist", "logits", "alphas", "logp", "xh", "call", "gates", "out2", "ctx"):
                if k in F:
                    assert torch.equal(F[k].view(torch.uint8), again[-1][k].view(torch.uint8)), "deterministic: two runs differ"
    for k, v in ck.worst.items():
        _WORST["tf " + k] = max(_WORST.get("tf " + k, 0.0), v)
    _INSIDE[case] = max(_INSIDE.get(case, 0), inside)
    print("\n%-34s decisions inside the margin %d  %s" % (ck.tag, inside,
                                                        "  ".join("%s %.3f" % kv for kv in sorted(ck.worst.items()))))


def test_zz_worst_ratios():
    """Prints the worst |y - ref| / bound per quantity over the cases above (run after them)."""
    if not _WORST:
        pytest.skip("run with the step tests")
    print("\nworst |y - ref| / bound per quantity:")
    for k, v in sorted(_WORST.items()):
        print("  %-28s %.4f" % (k, v))
    print("decisions inside the fp32 margin per case: %s" % _INSIDE)
