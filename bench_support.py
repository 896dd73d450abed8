"""Helpers for bench.py: synthetic workload, per-kernel roofline probes (CUDA events on the launching
stream), launch counting, and the CPU baseline leg (the only place outside tests/ that runs oracle/)."""
import ctypes
import os
import time

import torch


def tc_ready():
    from latex_ocr_b200 import _lib
    return bool(_lib.lib().lo_tc_available())


def synthetic_batch(B, H, W, V, T, seed):
    """SURVEY.md §8-d: white (255) background with 10 % random ink; targets of length U{20..T}, then END,
    PAD up to T+1 columns (model/utils/text.py:157-162).  ids 0..V-4 tokens, V-2 PAD, V-1 END."""
    g = torch.Generator().manual_seed(seed)
    img = torch.full((B, 1, H, W), 255.0)
    ink = torch.rand((B, 1, H, W), generator=g) < 0.10
    img = torch.where(ink, torch.randint(0, 255, (B, 1, H, W), generator=g).float(), img)
    lens = torch.randint(min(20, T), T + 1, (B,), generator=g)
    lens[0] = T
    formula = torch.full((B, T + 1), V - 2, dtype=torch.long)
    for b in range(B):
        n = int(lens[b])
        formula[b, :n] = torch.randint(0, V - 3, (n,), generator=g)
        formula[b, n] = V - 1
    return img, formula


DUMP_SAMPLE = 1 << 20     # parameters larger than this are dumped as a fixed sample: a dump of either workload stays < 64 MB


def step_outputs(model, loss):
    """Host copies of what one train step hands its caller: the loss vector [total, ce, reg, n_valid] (float64) and every
    parameter after the step's Adam update (float32; tensors above DUMP_SAMPLE elements as a fixed, seeded sample of
    their flattened values).  Taken right after the timed steps, before anything else updates the parameters."""
    out = {"loss": loss.detach().double().cpu().numpy()}
    for mod in ("encoder", "decoder", "row_encoder", "layer2"):
        m = getattr(model, mod, None)
        if m is None:
            continue
        for name, t in m.state_dict().items():
            flat = t.detach().float().reshape(-1)
            if flat.numel() > DUMP_SAMPLE:
                idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:DUMP_SAMPLE].sort().values
                flat = flat[idx.to(flat.device)]
            out["%s.%s" % (mod, name)] = flat.cpu().numpy()
    return out


def write_outputs(directory, arrays):
    import numpy as np
    os.makedirs(directory, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(directory, name + ".npy"), a)


def launches_per_step(model, img_dev, formula_dev):
    """Kernels launched by ONE train step (counted on an eager replay of the same step body)."""
    from latex_ocr_b200 import _lib
    N, L = formula_dev.shape
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    mask = model.decoder.make_dropout_mask(N, L - 1)
    model._step_body(img_dev.float(), formula_dev, [L - 1] * N, mask)
    torch.cuda.synchronize()
    return _lib.launch_count() - n0


def _time_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_probes(model, c, pk):
    """Roofline objects for the two kernels the north star names:
       attention step kernel — HBM bound: algorithmic bytes = B*R*(A+C)*bpe + B*R*4 per launch (SURVEY §8-d)
       conv stack fwd+bwd   — tensor bound: 56.0 GFLOP per image (fwd + dgrad + wgrad)."""
    from latex_ocr_b200 import _lib
    L = _lib.lib()
    dec, enc = model.decoder, model.encoder
    B, T = c["B"], c["T"]
    key = [k for k in dec._ws if k[0] == B and k[1] == T][0]
    R = key[2]
    ws = dec._ws[key]
    t, a = ws["t"], ws["args"]
    bpe = 2 if dec.precision == "bf16" else 4
    A = C = 512
    O1 = A + C + 4 * 512
    enc_ws = enc._ws[(B, c["H"], c["W"])]
    enc_out = enc_ws["out"].view(B, R, C)
    st = _lib.stream_ptr()
    dt = _lib.LO_BF16 if bpe == 2 else _lib.LO_F32

    def att_steps():
        for s in range(T):
            o1 = t["out1"][s]
            _lib.check(L.lo_attention_forward(_lib.ptr(t["att1"]), _lib.ptr(enc_out), dt, _lib.ptr(o1), O1, a.w_full,
                                              ctypes.c_void_p(t["alphas"].data_ptr() + s * R * 4), T * R, _lib.ptr(t["ctx"][s]),
                                              None, 0, None, B, R, A, C, _lib.ptr(t["work"]), st))

    mask_step = t["att_mask"][0]          # [B][R][A/8] bits of one step (any step's bits give the same traffic)

    def att_steps_mask():
        for s in range(T):
            o1 = t["out1"][s]
            _lib.check(L.lo_attention_forward_mask(_lib.ptr(t["att1"]), _lib.ptr(enc_out), dt, _lib.ptr(o1), O1, a.w_full,
                                                   ctypes.c_void_p(t["alphas"].data_ptr() + s * R * 4), T * R, _lib.ptr(t["ctx"][s]),
                                                   None, 0, None, _lib.ptr(t["att_mask"][s]), B, R, A, C, _lib.ptr(t["work"]), st))

    maskbits = bool(_lib.lib().lo_get_option(b"att_maskbits"))
    # the stand-alone attention entry points are launched without programmatic dependent launch unless the caller vouches for the age
    # of the tensors they read early; here those are static, and the time loop launches its attention kernels WITH the overlap
    _lib.set_option("att_abi_pdl", 1)
    ms_att = _time_ms(att_steps_mask if maskbits else att_steps, 3) / T
    att_bytes = B * R * (A + C) * bpe + B * R * 4 + (B * R * A // 8 if maskbits else 0)
    att = {"kernel": "attention_fwd_pipe_kernel (score + softmax + context + gate, one decode step, TMA ring)", "bound": "hbm",
           "achieved": att_bytes / (ms_att * 1e-3) / 1e9, "peak": pk["hbm"], "unit": "GB/s", "traffic": None,
           "us_per_launch": ms_att * 1e3, "algorithmic_bytes": att_bytes, "peak_source": pk["src"]}
    att["frac"] = att["achieved"] / att["peak"]

    # attention backward step kernel: the same stream (att1 + enc read once) + the d e row written
    DX = C + 512

    def att_bwd_steps():
        for s in range(T - 1, -1, -1):
            o1 = t["out1"][s]
            _lib.check(L.lo_attention_backward(_lib.ptr(t["att1"]), _lib.ptr(enc_out), dt, _lib.ptr(o1), ctypes.c_void_p(o1.data_ptr() + A * 4), O1,
                                               a.w_full, ctypes.c_void_p(t["alphas"].data_ptr() + s * R * 4), T * R, _lib.ptr(t["ctx"][s]),
                                               _lib.ptr(t["dxh"]), DX, _lib.ptr(t["dreg"]), R, ctypes.c_void_p(t["sreg"].data_ptr() + s * 4), T,
                                               ctypes.c_void_p(t["de"].data_ptr() + s * R * 4), _lib.ptr(t["dcat"][s]),
                                               ctypes.c_void_p(t["dcat"][s].data_ptr() + A * 4), O1, _lib.ptr(t["dctx"][s]), None,
                                               _lib.ptr(t["att_mask"][s]) if maskbits else None, B, R, A, C, _lib.ptr(t["work"]), st))

    ms_attb = _time_ms(att_bwd_steps, 3) / T
    _lib.set_option("att_abi_pdl", 0)
    # algorithmic bytes of the backward: enc read once + 1 mask bit per att1 element (or att1 itself without the mask scheme)
    # + alpha read and d e written
    attb_bytes = (B * R * C * bpe + B * R * A // 8 + 2 * B * R * 4) if maskbits else att_bytes
    mma = maskbits and bool(_lib.lib().lo_get_option(b"att_bwd_mma")) and bpe == 2
    kname = ("attention_bwd_mma_kernel" if mma else "attention_bwd_mask_kernel") if maskbits else "attention_bwd_pipe_kernel"
    attb = {"kernel": kname + " (d alpha, softmax backward, ReLU-mask sums, one decode step, TMA ring"
                      + ("; streams enc + the forward's mask bits instead of enc + att1" if maskbits else "")
                      + ("; both contractions on mma.sync)" if mma else ")"), "bound": "hbm",
            "achieved": attb_bytes / (ms_attb * 1e-3) / 1e9, "peak": pk["hbm"], "unit": "GB/s",
            "traffic": None, "us_per_launch": ms_attb * 1e3, "algorithmic_bytes": attb_bytes,
            "peak_source": pk["src"]}
    attb["frac"] = attb["achieved"] / attb["peak"]

    img = enc_ws["img"]
    denc = t["denc"].view(B, enc_ws["out"].shape[1], enc_ws["out"].shape[2], C)

    def conv_all():
        enc.forward_raw(img, need_grad=True)
        enc.backward_raw(tuple(img.shape), denc)

    ms_conv = _time_ms(conv_all, 3)
    flops = B * 56.0e9
    conv = {"kernel": "conv stack fwd+dgrad+wgrad (6 layers, incl. pools/ReLU masks)", "bound": "tensor",
            "achieved": flops / (ms_conv * 1e-3) / 1e12, "peak": pk["tf_sustained"], "unit": "TFLOP/s", "traffic": None,
            "ms": ms_conv, "algorithmic_flops": flops, "peak_source": pk["src"]}
    conv["frac"] = conv["achieved"] / conv["peak"]

    # the wgmma kernels alone (layers 2-6: forward, data gradient, weight gradient) — what SURVEY §8-d calls the tensor-pipe
    # figure (conv1 / pools / masks / bias-gradient column sums are memory-bound CUDA-core kernels and are excluded here)
    from latex_ocr_b200.encoder import _LAYERS
    Aa, Gg, S = enc_ws["acts"], enc_ws["grads"], enc.store
    impl = enc._impl()
    cfgl = {l[0]: l for l in _LAYERS}
    plan = (("14", "P11"), ("11", "P8"), ("8", "Y6"), ("6", "P3"), ("3", "P0"))
    fwd_in = {"3": "P0", "6": "P3", "8": "Y6", "11": "P8", "14": "P11"}

    def conv_tc():
        for idx, cin, cout, pad, pool in _LAYERS[1:]:
            x = Aa[fwd_in[idx]]
            _lib.check(L.lo_conv3x3(_lib.ptr(x), _lib.ptr(S.w("cnn.%s.weight" % idx)), _lib.ptr(S.f32("cnn.%s.bias" % idx)), None,
                                    _lib.ptr(Aa["Y" + idx]), dt, B, x.shape[1], x.shape[2], cin, cout, pad, 1, impl, st))
        for idx, xin in plan:
            _, cin, cout, pad, pool = cfgl[idx]
            x, dy = Aa[xin], Gg["Y" + idx]
            # db = NULL: the bias-gradient column sums are memory-bound CUDA-core kernels, not part of the tensor-pipe figure
            _lib.check(L.lo_conv3x3_wgrad(_lib.ptr(x), _lib.ptr(dy), _lib.ptr(S.g("cnn.%s.weight" % idx)), None,
                                          dt, B, x.shape[1], x.shape[2], cin, cout, pad, impl, st))
            mask = Aa[xin] if xin.startswith("Y") else None
            _lib.check(L.lo_conv3x3(_lib.ptr(dy), _lib.ptr(enc_ws["wflip"][idx]), None, _lib.ptr(mask), _lib.ptr(Gg[xin]), dt, B, dy.shape[1],
                                    dy.shape[2], cout, cin, 2 - pad, 0, impl, st))

    ms_tc = _time_ms(conv_tc, 3)
    flops_tc = B * 3 * 2 * 9.296e9     # layers 2-6: 9.296 GMAC/image, x3 passes (fwd, dgrad, wgrad)
    conv_tc_r = {"kernel": "wgmma conv kernels only: tc_conv_p_kernel (persistent, 128x256 tiles, fwd + dgrad) and tc_wgrad_kernel, "
                           "layers 2-6 (15 launches)", "bound": "tensor",
                 "achieved": flops_tc / (ms_tc * 1e-3) / 1e12, "peak": pk["tf_sustained"], "unit": "TFLOP/s",
                 "traffic": None, "ms": ms_tc,
                 "algorithmic_flops": flops_tc, "peak_source": pk["src"]}
    conv_tc_r["frac"] = conv_tc_r["achieved"] / conv_tc_r["peak"]

    def dec_all():
        _lib.check(L.lo_decoder_forward(ctypes.byref(a), 1, st))
        _lib.check(L.lo_decoder_backward(ctypes.byref(a), st))

    ms_dec = _time_ms(dec_all, 2)
    extra = {"decoder_fwd_bwd_ms": ms_dec, "encoder_fwd_bwd_ms": ms_conv, "attention_fwd_us_per_step": ms_att * 1e3,
             "attention_bwd_us_per_step": ms_attb * 1e3}
    # the dominant kernel = the largest MEASURED share of the step among the kernels the north star names
    share = {"attention_fwd": T * ms_att, "attention_bwd": T * ms_attb, "conv_tensor_kernels": ms_tc}
    extra["kernel_share_ms"] = share
    dominant = {"attention_fwd": att, "attention_bwd": attb, "conv_tensor_kernels": conv_tc_r}[max(share, key=share.get)]
    return {"dominant": dominant, "all": {"attention": att, "attention_bwd": attb, "conv": conv, "conv_tensor_kernels": conv_tc_r,
                                          "phases": extra}}


def cpu_threads():
    """Threads for the CPU arm: every core the process may use (affinity and cgroup quota respected), capped by
    LO_CPU_THREADS.  Oversubscribing a quota-limited container makes the OpenMP barriers of the 150-step loop crawl."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = max(1, min(n, int(int(q) / int(p))))
    except Exception:
        pass
    return max(1, min(n, int(os.environ.get("LO_CPU_THREADS", "64"))))


def cpu_arm(c, sample_b, steps, warmup):
    """Times the reference's CPU train step (getLoss: forward, loss, backward, two Adam steps — img2seq_torch.py:136-172) on
    `sample_b` images of the cfg2 workload, all host threads.  When the reference tree is importable (/root/reference in the
    build container, baseline/_ref on a box where the driver installed it) the UNMODIFIED reference modules are driven through
    oracle/ref_shim.py (kind "reference"); otherwise the oracle port executes the same un-hoisted algorithm (kind "port").
    Returns (seconds per step, kind, cores)."""
    from oracle import ref_model as rm
    from oracle import ref_shim
    cores = cpu_threads()
    torch.set_num_threads(cores)
    img, formula = rm.synthetic_batch(sample_b, c["H"], c["W"], c["V"], c["T"], c["T"], seed=1234)
    T = formula.shape[1] - 1
    if ref_shim.reference_available():
        kind = "reference"
        enc, dec = ref_shim.build_reference_models(c["V"])
        enc.train(True)
        dec.train(True)                                            # nn.Dropout(0.5) active, as in the reference's training loop
        oe = torch.optim.Adam(enc.parameters(), lr=1e-3)          # img2seq_torch.py:86-87
        od = torch.optim.Adam(dec.parameters(), lr=1e-3)

        def step():
            loss, _, _ = ref_shim.ref_get_loss(enc, dec, img, formula)
            od.zero_grad()
            oe.zero_grad()
            loss.backward()
            od.step()
            oe.step()
            return loss.item()
    else:
        kind = "port"
        pe, pd = rm.init_params(c["V"], seed=0)
        state = {}
        gen = torch.Generator().manual_seed(7)

        def step():
            mask = (torch.rand(sample_b, T, 512, generator=gen) >= 0.5).float() * 2.0
            return rm.train_step(pe, pd, img, formula, state, dropout_mask=mask, hoist=False)[0]
    for _ in range(warmup):
        step()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    return (time.perf_counter() - t0) / steps, kind, cores


def cpu_baseline(c):
    """`cpu_baseline` of the product arm's JSON line: the reference's CPU algorithm on this box's host cores, on a bounded
    sample of the workload (same sample size as `bench.py --impl reference`)."""
    sb = int(os.environ.get("LO_REF_SAMPLE_B", "8"))
    dt, kind, cores = cpu_arm(c, sb, steps=2, warmup=1)
    return {"value": sb / dt, "unit": "images/s", "cores": cores, "kind": kind,
            "sample": "%d of %d images per step (cfg2 shapes), 2 timed steps after 1 warm-up, torch %s CPU fp32, %.2f s/step"
                      % (sb, c["B"], torch.__version__, dt)}


def decode_probe(model, V=500, n_images=256, height=64, widths=(64, 128, 256, 512, 1024), max_len=150, beam=5, oracle_sample=True):
    """BASELINE.json configs[4] (cfg #5): greedy and beam-5 decoding of `n_images` variable-width images through the public
    ``Img2SeqModel.predict_batch`` with HOST uint8 images (list of HxWx1 arrays -> shape bucketing like
    utils/data_generator.py:84-122 -> pad -> H2D -> encoder -> decode loop -> ids D2H -> truncate), bf16 storage.
    Random-init weights never emit END, so every batch runs the full max_length_formula + 2 = 152 steps; tokens/s counts the
    tokens of the scored hypothesis (hypothesis 0, img2seq.py:210).  `exact_match_vs_oracle`: the fp32 CPU oracle's greedy
    decode (oracle/ref_decode.py) of a bounded sample (2 images per bucket, 24 steps) against the GPU bf16 ids."""
    import numpy as np
    from latex_ocr_b200 import data as lod
    rng = np.random.RandomState(5)
    per = n_images // len(widths)
    imgs = []
    for i, W in enumerate(widths):
        n = per + (n_images - per * len(widths) if i == len(widths) - 1 else 0)
        for _ in range(n):
            a = np.full((height, W, 1), 255, np.uint8)
            ink = rng.rand(height, W, 1) < 0.10
            a[ink] = rng.randint(0, 255, size=int(ink.sum())).astype(np.uint8)
            imgs.append(a)
    order = rng.permutation(len(imgs))
    items = lod.bucket_by_shape([(imgs[i], int(i)) for i in order], per)          # same-shape runs of `per` images
    batches = [[it[0] for it in items[k:k + per]] for k in range(0, len(items), per)]
    batches = [b for b in batches if b]
    cfgd = model._config
    # one workspace per (bucket, mode) must stay cached NEXT TO whatever the training part of the run left in the bounded caches:
    # one entry too few and the LRU order makes every batch of the timed pass re-allocate its workspace (observed: beam-5 at a third
    # of its rate)
    model.decoder._ws.maxsize = len(model.decoder._ws) + 2 * len(widths) + 4
    model.encoder._ws.maxsize = len(model.encoder._ws) + 2 * len(widths) + 4
    out = {"workload": "cfg5: %d images %d x {%s} px, bucketed by width (batches of %d), %d decode steps, bf16, host uint8 images in, "
                       "token ids out; faster of two timed passes after one warm-up pass" % (n_images, height, ",".join(map(str, widths)), per, max_len + 2)}
    for mode, bs in (("greedy", 1), ("beam5", beam)):
        cfgd.decoding = "greedy" if bs == 1 else "beam_search"
        cfgd.beam_size = bs
        cfgd.max_length_formula = max_len
        dt = None
        for rep in range(3):                                                         # first pass warms the per-bucket workspaces;
            torch.cuda.synchronize()                                                 # the faster of the two timed passes is reported
            t0 = time.perf_counter()
            toks = 0
            for b in batches:
                ids, _ = model._decode_ids(torch.from_numpy(lod.pad_batch_images(b)).permute(0, 3, 1, 2).contiguous())
                toks += sum(len(s) for s in ids[0])
            torch.cuda.synchronize()
            if rep > 0:
                dt = time.perf_counter() - t0 if dt is None else min(dt, time.perf_counter() - t0)
        out[mode + "_tok_s"] = toks / dt
        out[mode + "_img_s"] = n_images / dt
        out[mode + "_seconds"] = dt
    if oracle_sample:
        from oracle import ref_decode as rd
        from oracle import ref_model as rm
        pe = {k: v.detach().float().cpu() for k, v in model.encoder.state_dict().items()}
        pd = {k: v.detach().float().cpu() for k, v in model.decoder.state_dict().items()}
        steps, match, total, exact, nseq = 24, 0, 0, 0, 0
        cfgd.decoding, cfgd.max_length_formula = "greedy", steps - 2
        for W in widths:
            b = [im for im in imgs if im.shape[1] == W][:2]
            x = torch.from_numpy(lod.pad_batch_images(b)).permute(0, 3, 1, 2).contiguous()
            enc = rm.encoder_forward(pe, x.float()).reshape(len(b), -1, 512)
            want = rd.greedy_decode(pd, enc, start_id=V - 2, end_id=V - 1, max_iter=steps - 1)
            got, _ = model._decode_ids(x)
            got = torch.tensor(got[0])[:, :want.shape[1]]
            match += int((got == want[:, :got.shape[1]]).sum())
            total += got.numel()
            exact += int((got == want[:, :got.shape[1]]).all(dim=1).sum())
            nseq += len(b)
        out["exact_match_vs_oracle"] = exact / max(nseq, 1)
        out["token_match_vs_oracle"] = match / max(total, 1)
        out["oracle_sample"] = "%d images (2 per width bucket), %d free-running greedy steps, fp32 CPU oracle vs bf16 GPU" % (nseq, steps)
    cfgd.max_length_formula = max_len
    return out
