"""Greedy / beam-search decoding on the H100 step kernels — the decode row of SURVEY.md §8 (a8).

Loop semantics follow the reference's TF decode loop, which is framework independent:
  dynamic_decode (model/components/dynamic_decode.py:38-61): run until every row is finished, at most
  max_length_formula + 2 steps (``finished |= time >= max_iter`` with max_iter = max_length_formula + 1, decoder.py:70);
  greedy (greedy_decoder_cell.py:53-66): id = argmax, finished |= id == END, rows keep decoding after END;
  beam (beam_search_decoder_cell.py:123-250): see include/latex_ocr_b200.h:lo_decoder_beam; ``finalize='reference'``
  reproduces the reference's identity finalize (its back-tracking loop never updates ``parents``, :237), ``'backtrack'``
  returns lineage-consistent hypotheses.
The torch flavour of the reference has no START symbol; the caller supplies ``start_id`` (SURVEY.md §8-c).

``img`` is a tensor [N,1,H,W] (one size for the batch) or a list of images of different sizes, each a [1,H,W] tensor or an HxWx1
uint8 array.  A list is decoded in ONE time loop in which every image attends over its own regions only (lo_decoder_args.reg_off):
no padding, and an image's tokens are those it gets when decoded alone.
"""
import collections
import ctypes

import torch

from . import _lib
from ._lib import check, stream_ptr


def _n_steps(fin_hist):
    """fin_hist [N, steps(, beam)] int32 -> number of loop iterations the reference would have executed."""
    N = fin_hist.shape[0]
    S = fin_hist.shape[1]
    allf = fin_hist.reshape(N, S, -1).all(dim=2).all(dim=0)          # [S]
    idx = torch.nonzero(allf)
    return int(idx[0]) + 1 if idx.numel() else S


def _prepare(model, img, rows_per_img, max_steps):
    enc = model.encoder.forward_raw(img.to(model.device).float(), need_grad=False)
    N = enc.shape[0]
    R = enc.shape[1] * enc.shape[2]
    enc_flat = enc.view(N, R, enc.shape[3])
    dec = model.decoder
    B = N * rows_per_img
    ws = dec.workspace(B, max_steps, R, need_grad=False)
    dec.store.refresh_shadow()
    for t in range(max_steps):
        ws["bt"][t] = B
    a = dec.fill_args(ws, enc_flat, B, max_steps, R, has_dropout=False)
    a.rows_per_img = rows_per_img
    return a, ws, N


def _image(x):
    """one image of a list: [1,H,W] tensor (uint8 or float) on the CPU or the GPU"""
    t = x if torch.is_tensor(x) else torch.from_numpy(x).permute(2, 0, 1)      # HxWx1 array -> [1,H,W]
    if t.dim() != 3 or t.shape[0] != 1:
        raise ValueError("each image must be a [1,H,W] tensor or an HxWx1 array (got shape %s)" % (tuple(t.shape),))
    return t


RaggedLayout = collections.namedtuple("RaggedLayout", ("imgs", "order", "groups", "counts", "off"))


def ragged_layout(images, out_hw):
    """Decode order and packed layout of a list of images of different sizes (both flavours).  The images are sorted by shape so
    that the encoder runs once per distinct shape and each run's output (a workspace buffer the next run overwrites) is one
    contiguous copy into the packed enc.  ``out_hw(H, W)``: the encoder's feature-map size.  Returns a RaggedLayout: the images as
    [1,H,W] tensors in input order; order[j] = the input index of decode image j; groups = [first, end) runs of one shape in decode
    order; counts[j] = the region count of decode image j; off = their prefix offsets (reg_off)."""
    imgs = [_image(x) for x in images]
    if not imgs:
        raise ValueError("no images")
    order = sorted(range(len(imgs)), key=lambda i: tuple(imgs[i].shape[1:]))
    groups = []                                          # [first, end) runs of one shape in decode order
    for j, i in enumerate(order):
        if groups and tuple(imgs[order[groups[-1][0]]].shape[1:]) == tuple(imgs[i].shape[1:]):
            groups[-1][1] = j + 1
        else:
            groups.append([j, j + 1])
    counts = []
    for j0, j1 in groups:
        h, w = out_hw(*imgs[order[j0]].shape[1:])
        counts += [h * w] * (j1 - j0)
    if min(counts) < 1:
        raise ValueError("an image is too small for the encoder (no feature-map region)")
    off = [0]
    for n in counts:
        off.append(off[-1] + n)
    return RaggedLayout(imgs, order, groups, counts, off)


def encode_packed(encoder, lay, enc, device):
    """Runs ``encoder`` once per shape group of ``lay`` and writes its output into the packed ``enc`` [regions, C] in decode
    order."""
    imgs, order, off = lay.imgs, lay.order, lay.off
    for j0, j1 in lay.groups:
        batch = torch.stack([imgs[order[j]] for j in range(j0, j1)]).to(device)
        e = encoder.forward_raw(batch if batch.dtype == torch.uint8 else batch.float(), need_grad=False)
        enc[off[j0]:off[j1]].copy_(e.reshape(off[j1] - off[j0], e.shape[3]))


def _prepare_ragged(model, images, rows_per_img, max_steps):
    """Packed encoder output and the argument block of a decode over images of different sizes (ragged_layout).  Returns (args,
    workspace, order, region counts) with order[j] = the input index of decode image j."""
    lay = ragged_layout(images, model.encoder.out_hw)
    order, counts, off = lay.order, lay.counts, lay.off
    N, R, dev, dec = len(order), max(counts), model.device, model.decoder
    B = N * rows_per_img
    ws = dec.ragged_workspace(B, max_steps, R, off[-1])
    encode_packed(model.encoder, lay, ws["t"]["enc"], dev)
    host = ws["reg_off_host"]
    for i, v in enumerate(off):
        host[i] = v
    ws["t"]["reg_off"][:N + 1].copy_(torch.tensor(off, dtype=torch.int32))
    dec.store.refresh_shadow()
    for t in range(max_steps):
        ws["bt"][t] = B
    a = dec.fill_args(ws, ws["t"]["enc"], B, max_steps, R, has_dropout=False)
    a.rows_per_img = rows_per_img
    a.reg_off = ws["t"]["reg_off"].data_ptr()
    a.reg_off_host = ctypes.cast(host, ctypes.c_void_p)
    return a, ws, order, counts


def _inverse(order):
    inv = [0] * len(order)
    for j, i in enumerate(order):
        inv[i] = j
    return torch.tensor(inv, dtype=torch.int64)


def greedy_decode(model, img, start_id, end_id, max_length_formula=150, return_attention=False):
    """Returns token ids [N, steps] (CPU int64), steps as the reference's loop would have run.  ``return_attention=True`` also
    returns the attention weights of every step, [N, steps, R] fp32 on the CPU — what the reference collects in
    ``attention_mechanism.ctx_vector`` for visualize_attention.py (attention_mechanism.py:96-121).  For a list of images the ids
    are in input order and the attention weights are a list of [steps, R_i] tensors, R_i the image's own region count."""
    L = _lib.lib()
    max_steps = max_length_formula + 2
    with torch.no_grad():
        if isinstance(img, (list, tuple)):
            a, ws, order, counts = _prepare_ragged(model, img, 1, max_steps)
            N = len(order)
        else:
            a, ws, N = _prepare(model, img, 1, max_steps)
        dev = model.device
        tokens = torch.zeros(N, max_steps, dtype=torch.int64, device=dev)
        finished = torch.zeros(N, dtype=torch.int32, device=dev)
        hist = torch.zeros(N, max_steps, dtype=torch.int32, device=dev)
        check(L.lo_decoder_greedy_hist(ctypes.byref(a), int(start_id), int(end_id), max_steps, tokens.data_ptr(), finished.data_ptr(),
                                       hist.data_ptr(), stream_ptr()))
        n = _n_steps(hist.cpu())
        if isinstance(img, (list, tuple)):
            inv = _inverse(order)
            ids = tokens[:, :n].cpu()[inv]
            if return_attention:
                al = ws["t"]["alphas"].view(-1)[:N * max_steps * a.R].view(N, max_steps, a.R)[:, :n].cpu()
                return ids, [al[j, :, :counts[j]].clone() for j in inv.tolist()]
            return ids
        if return_attention:
            return tokens[:, :n].cpu(), ws["t"]["alphas"][:, :n].float().cpu()
        return tokens[:, :n].cpu()


def attention_maps(alphas, att_h, att_w):
    """visualize_attention.py:49-72 (getOutArray): an attention vector over the R = att_h * att_w regions as a grey image,
    region r at (r // att_w, r % att_w), value (1 - alpha) * 255 (dark = attended).  alphas [..., R] -> float [..., att_h, att_w]."""
    a = torch.as_tensor(alphas, dtype=torch.float32)
    if a.shape[-1] != att_h * att_w:
        raise ValueError("attention vector of %d regions does not match a %dx%d feature map" % (a.shape[-1], att_h, att_w))
    return ((1.0 - a) * 255.0).reshape(tuple(a.shape[:-1]) + (att_h, att_w))


def beam_decode(model, img, start_id, end_id, beam_size=5, max_length_formula=150, finalize="reference",
                div_gamma=1, div_prob=0, div_u=None, div_seed=None):
    """Returns (ids [N, beam, steps], log_probs [N, beam]) on the CPU; hypothesis 0 is the one the reference scores
    (img2seq.py:210).  ``div_gamma`` / ``div_prob``: the diversity penalty of beam_search_decoder_cell.py:258-287 (off when
    gamma == 1 or prob == 0, as in configs/model.json:15-16); its Bernoulli draws come from the in-kernel Philox stream seeded
    by ``div_seed`` (default: torch's initial seed), or from ``div_u`` — uniforms [steps, N*beam, V] — when given (tests).  For a
    list of images, results are in input order and image i draws the rows [i*beam, (i+1)*beam) of ``div_u``."""
    if finalize not in ("reference", "backtrack"):
        raise NotImplementedError("finalize must be 'reference' or 'backtrack'")
    L = _lib.lib()
    max_steps = max_length_formula + 2
    ragged = isinstance(img, (list, tuple))
    with torch.no_grad():
        if ragged:
            a, ws, order, _ = _prepare_ragged(model, img, beam_size, max_steps)
            N = len(order)
        else:
            a, ws, N = _prepare(model, img, beam_size, max_steps)
        dev = model.device
        ids = torch.zeros(N, max_steps, beam_size, dtype=torch.int64, device=dev)
        parents = torch.zeros_like(ids)
        hist = torch.zeros(N, max_steps, beam_size, dtype=torch.int32, device=dev)
        logp = torch.zeros(N, beam_size, dtype=torch.float32, device=dev)
        div_on = not (div_gamma == 1 or div_prob == 0)
        u_dev = state = None
        if div_on and div_u is not None:
            u_dev = torch.as_tensor(div_u, dtype=torch.float32).to(dev).contiguous()
            if tuple(u_dev.shape) != (max_steps, N * beam_size, a.V):
                raise ValueError("div_u must be [max_length_formula + 2, N * beam, V]")
            if ragged:          # decode order
                u_dev = u_dev.view(max_steps, N, beam_size, a.V)[:, torch.tensor(order, device=dev)].reshape(max_steps, N * beam_size, a.V)
        elif div_on:
            seed = torch.initial_seed() if div_seed is None else int(div_seed)
            state = torch.tensor([seed & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64, device=dev)
        check(L.lo_decoder_beam_div(ctypes.byref(a), int(start_id), int(end_id), max_steps, ids.data_ptr(), parents.data_ptr(),
                                    hist.data_ptr(), logp.data_ptr(), float(div_gamma), float(div_prob),
                                    u_dev.data_ptr() if u_dev is not None else None,
                                    state.data_ptr() if state is not None else None, stream_ptr()))
        n = _n_steps(hist.cpu())
        ids, parents, logp = ids[:, :n].cpu(), parents[:, :n].cpu(), logp.cpu()
        if ragged:
            inv = _inverse(order)
            ids, parents, logp = ids[inv], parents[inv], logp[inv]
        if finalize == "backtrack":
            out = torch.zeros_like(ids)
            cur = torch.arange(beam_size).unsqueeze(0).repeat(N, 1)
            for t in range(n - 1, -1, -1):
                out[:, t] = torch.gather(ids[:, t], 1, cur)
                cur = torch.gather(parents[:, t], 1, cur)
            ids = out
        return ids.permute(0, 2, 1).contiguous(), logp      # [N, beam, time] like img2seq.py:239-241


def truncate_end(list_of_ids, id_end):
    """model/evaluation/text.py:95-104."""
    out = []
    for seq in list_of_ids:
        seq = [int(t) for t in seq]
        out.append(seq[:seq.index(id_end)] if id_end in seq else seq)
    return out
