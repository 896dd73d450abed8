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

Also the host side both decoder flavours share (tf_decoder.Decoder): region offsets, the ragged workspace's capacity rule, and
greedy / beam calls with their outputs trimmed to the steps the reference would have run.
"""
import collections
import ctypes
import itertools
import math

import torch

from . import _lib
from ._lib import check, stream_ptr
from .kernel_module import stamp


def _n_steps(fin_hist):
    """fin_hist [N, steps(, beam)] int32 -> number of loop iterations the reference would have executed."""
    N = fin_hist.shape[0]
    S = fin_hist.shape[1]
    allf = fin_hist.reshape(N, S, -1).all(dim=2).all(dim=0)          # [S]
    idx = torch.nonzero(allf)
    return int(idx[0]) + 1 if idx.numel() else S


def region_offsets(counts):
    """[0, n_0, n_0 + n_1, ...]: the offsets (reg_off) of images of ``counts`` regions, in decode order"""
    return list(itertools.accumulate((int(n) for n in counts), initial=0))


def set_region_offsets(a, host, dev, off):
    """Writes the offsets ``off`` into a ragged workspace's host array ``host`` and device tensor ``dev`` and points the args
    ``a`` (lo_decoder_args or lo_tfdec_args) at them."""
    for i, v in enumerate(off):
        host[i] = v
    dev[:len(off)].copy_(torch.tensor(off, dtype=torch.int32))
    a.reg_off = dev.data_ptr()
    a.reg_off_host = ctypes.cast(host, ctypes.c_void_p)


def ragged_cache(cache, cap, build):
    """The one ragged decode workspace of ``cache`` (key "ragged") for a call of capacity ``cap`` = (rows B, steps T, largest
    region count R, total regions).  A cached workspace whose capacity covers the call is reused; otherwise ``build(*cap)`` makes
    one of the element-wise maximum of both capacities (serving traffic gives a new composition on nearly every call)."""
    ws = cache.get("ragged")
    if ws is not None:
        if all(c <= h for c, h in zip(cap, ws["cap"])):
            return stamp(ws)
        cap = tuple(max(c, h) for c, h in zip(cap, ws["cap"]))
        del cache["ragged"]
    ws = build(*cap)
    ws["cap"] = cap
    cache["ragged"] = ws
    return ws


def run_greedy(call, N, steps, device):
    """Greedy decode of N rows: ``call(tokens, fin_hist)`` runs the flavour's entry point on the device pointers of the outputs
    [N, steps].  Returns the tokens [N, n] on the device, n the steps the reference would have run."""
    tokens = torch.zeros(N, steps, dtype=torch.int64, device=device)
    hist = torch.zeros(N, steps, dtype=torch.int32, device=device)
    check(call(tokens.data_ptr(), hist.data_ptr()))
    return tokens[:, :_n_steps(hist)]


def run_beam(call, N, beam, steps, V, device, div_u=None, order=None):
    """Beam search of N images: ``call(ids, parents, fin_hist, logp, div_u)`` runs the flavour's entry point on device pointers.
    ``div_u``: None or injected uniforms [steps, N * beam, V] in input order (``order``: the input index of each decode image).
    Returns (ids [N, n, beam], parents [N, n, beam], logp [N, beam]) on the device, n the steps the reference would have run."""
    ids = torch.zeros(N, steps, beam, dtype=torch.int64, device=device)
    parents = torch.zeros_like(ids)
    hist = torch.zeros(N, steps, beam, dtype=torch.int32, device=device)
    logp = torch.zeros(N, beam, dtype=torch.float32, device=device)
    if div_u is not None:
        div_u = torch.as_tensor(div_u, dtype=torch.float32).to(device).contiguous()
        if tuple(div_u.shape) != (steps, N * beam, V):
            raise ValueError("div_u must be [steps, N * beam, V] = [%d, %d, %d]" % (steps, N * beam, V))
        if order is not None:
            div_u = div_u.view(steps, N, beam, V)[:, torch.tensor(order, device=device)].reshape(steps, N * beam, V)
    check(call(ids.data_ptr(), parents.data_ptr(), hist.data_ptr(), logp.data_ptr(), div_u.data_ptr() if div_u is not None else None))
    n = _n_steps(hist)
    return ids[:, :n], parents[:, :n], logp


def penalty_weights(length_penalty, coverage_penalty):
    """(alpha, beta) of the length and coverage penalties of beam search as floats; a negative or non-finite weight is refused."""
    alpha, beta = float(length_penalty), float(coverage_penalty)
    for name, v in (("length_penalty", alpha), ("coverage_penalty", beta)):
        if not math.isfinite(v) or v < 0:
            raise ValueError("%s must be a finite number >= 0 (got %r)" % (name, v))
    return alpha, beta


def length_penalty_table(alpha, steps):
    """LP[l] = ((5 + l) / 6) ** alpha for l = 0..steps: the length penalty of GNMT (Wu et al. 2016, eq. 14) as TF's
    BeamSearchDecoder computes it (length_penalty_weight = alpha), in float64 and rounded once to fp32, so that the kernel and the
    CPU reference divide by the same numbers.  All ones for alpha = 0."""
    return (((5.0 + torch.arange(steps + 1, dtype=torch.float64)) / 6.0) ** float(alpha)).float()


def beam_penalty(alpha, beta, B, R, steps, beam, device):
    """The lo_beam_penalty of a beam search of B rows (B / beam images) over at most R regions and ``steps`` steps, and the tensors
    it points at, which must outlive the call: the length-penalty table, the coverage and length scratch, and ``scores`` [B / beam,
    beam], the winners' penalised scores after the last step."""
    t = {"len": torch.empty(2 * B, dtype=torch.int32, device=device),
         "scores": torch.zeros(B // beam, beam, dtype=torch.float32, device=device)}
    if alpha != 0:
        t["len_pen"] = length_penalty_table(alpha, steps).to(device)
    if beta > 0:
        t["cov"] = torch.empty(2 * B * R + B, dtype=torch.float32, device=device)     # [2][B][R] coverage, then [B] terms
    p = _lib.BeamPenalty()
    p.alpha, p.beta = alpha, beta
    for k in ("len_pen", "cov", "len", "scores"):
        setattr(p, k, t[k].data_ptr() if k in t else None)
    return p, t


def beam_hypotheses(ids, parents, finalize, a=None, alphas=None):
    """The hypotheses of run_beam's ``ids`` / ``parents`` [N, n, beam] (device) as ids [N, beam, n] and, with ``alphas``, their
    attention weights [N, beam, n, R] (lo_beam_backtrack), both on the device.  ``finalize``: 'reference' (slot s of every step, the
    reference's identity finalize) or 'backtrack' (the lineage of the final slot s).  ``alphas``: the decode's attention rows [B, T, R]
    (row b = image b // beam, slot b % beam); ``a``: the decode's args, whose region offsets (reg_off) give each image's own count
    (entries past it are 0).  Returns (ids, attention or None)."""
    N, n, beam = ids.shape
    out = torch.empty(N, beam, n, dtype=torch.int64, device=ids.device)
    att = None
    if alphas is not None:
        att = torch.empty(N, beam, n, alphas.shape[2], dtype=torch.float32, device=ids.device)
    mode = _lib.LO_BEAM_LINEAGE if finalize == "backtrack" else _lib.LO_BEAM_SLOTS
    check(_lib.lib().lo_beam_backtrack(ids.data_ptr(), parents.data_ptr(), ids.stride(0) // beam, N, beam, n,
                                       alphas.data_ptr() if att is not None else None, alphas.stride(0) if att is not None else 0,
                                       alphas.shape[2] if att is not None else 0, a.reg_off if a is not None else None,
                                       a.reg_off_host if a is not None else None, mode, out.data_ptr(),
                                       att.data_ptr() if att is not None else None, stream_ptr()))
    return out, att


class BracketRule:
    """Balanced brackets in decode (lo_bracket_rule): ``role[v]`` is 0 for a neutral token, +k for a token that opens kind k and
    -k for one that closes it.  Under a rule every greedy and sampled formula, and every beam hypothesis under
    ``finalize='backtrack'``, cut at its first END, nests the kinds properly, at most ``max_depth`` deep, and leaves none open
    (``check`` tells whether a sequence does).  The decode masks on the device, between the head and the token choice; the
    probabilities are the model's restricted to the allowed tokens.

    ``role``: V ints, each kind 1..n_kinds with at least one opening and one closing token (n_kinds = max |role|, at most 255);
    ``max_depth``: 1..32.  A table without kinds (all neutral) is accepted and changes nothing."""

    def __init__(self, role, max_depth=16):
        role = [int(r) for r in role]
        if not role:
            raise ValueError("empty role table")
        if not 1 <= int(max_depth) <= 32:
            raise ValueError("max_depth must lie in 1..32 (got %r)" % (max_depth,))
        bad = [v for v, r in enumerate(role) if not -255 <= r <= 255]
        if bad:
            raise ValueError("role of token %d out of range -255..255 (got %d)" % (bad[0], role[bad[0]]))
        self.n_kinds = max(abs(r) for r in role)
        for k in range(1, self.n_kinds + 1):
            if k not in role or -k not in role:
                raise ValueError("kind %d has no %s token" % (k, "opening" if k not in role else "closing"))
        self.role = role
        self.max_depth = int(max_depth)
        self._dev = {}

    @classmethod
    def latex(cls, id_to_tok, max_depth=16):
        """The rule of LaTeX formulas over a vocabulary (``id_to_tok``: a dict id -> token or a list): ``{`` / ``}`` are kind 1;
        every ``\\left`` + delimiter token (the character after ``\\left`` is not a letter, so ``\\leftarrow`` stays neutral) opens
        kind 2 and every ``\\right`` + delimiter token closes it, in any pairing (``\\left( ... \\right.`` is valid LaTeX); each
        ``\\begin{X}`` / ``\\end{X}`` pair of the vocabulary is a kind of its own (either without the other stays neutral).
        Everything else is neutral, ``\\{``, ``\\}``, parentheses and square brackets included."""
        toks = dict(id_to_tok) if isinstance(id_to_tok, dict) else dict(enumerate(id_to_tok))
        role = [0] * (max(toks) + 1)

        def delim(tok, cmd):
            return tok.startswith(cmd) and len(tok) > len(cmd) and not tok[len(cmd)].isalpha()

        def env(tok, cmd):
            return tok[len(cmd):-1] if tok.startswith(cmd) and tok.endswith("}") else None
        pairs = [([i for i, t in toks.items() if t == "{"], [i for i, t in toks.items() if t == "}"]),
                 ([i for i, t in toks.items() if delim(t, "\\left")], [i for i, t in toks.items() if delim(t, "\\right")])]
        for name in sorted({env(t, "\\begin{") for t in toks.values()} - {None}):
            pairs.append(([i for i, t in toks.items() if env(t, "\\begin{") == name],
                          [i for i, t in toks.items() if env(t, "\\end{") == name]))
        kind = 0
        for opens, closes in pairs:            # kinds in this order, a pair missing either side stays neutral
            if opens and closes:
                kind += 1
                for i in opens:
                    role[i] = kind
                for i in closes:
                    role[i] = -kind
        return cls(role, max_depth)

    def check(self, ids, end_id):
        """For every sequence of ``ids`` (a [..., steps] tensor or array, or a list of sequences), cut at its first ``end_id``:
        whether it nests properly, at most max_depth deep, and leaves no bracket open.  Returns a list of bools."""
        if torch.is_tensor(ids) or hasattr(ids, "shape"):
            t = torch.as_tensor(ids)
            seqs = t.reshape(-1, t.shape[-1]).tolist() if t.dim() >= 1 and t.numel() else []
        else:
            seqs = [list(s) for s in ids]
        end_id, V = int(end_id), len(self.role)
        out = []
        for seq in seqs:
            stack, ok = [], True
            for tok in seq:
                tok = int(tok)
                if tok == end_id:
                    break
                r = self.role[tok] if 0 <= tok < V else 0
                if r > 0:
                    stack.append(r)
                    ok = len(stack) <= self.max_depth
                elif r < 0:
                    ok = bool(stack) and stack.pop() == -r
                if not ok:
                    break
            out.append(ok and not stack)
        return out

    def device_role(self, device):
        """The role table as an int32 tensor on ``device``, copied once per device."""
        device = torch.device(device)
        if device not in self._dev:
            self._dev[device] = torch.tensor(self.role, dtype=torch.int32, device=device)
        return self._dev[device]

    def allowed_at_start(self, end_id, max_steps):
        """The tokens a row may take at step 0 of a call of ``max_steps`` steps (depth 0): END, neutral tokens and, with a step
        left to close them, opening ones."""
        return sum(1 for v, r in enumerate(self.role) if v == end_id or r == 0 or (r > 0 and max_steps >= 2))

    def args(self, end_id, V, B, max_steps, device, beam=1):
        """The lo_bracket_rule of a decode of B rows over V tokens and the tensors it points at, which must outlive the call.
        Refuses (ValueError) a table of another size than V, a non-neutral END and, for beam search, fewer tokens allowed at step 0
        than ``beam``."""
        if len(self.role) != V:
            raise ValueError("the rule's role table has %d entries, the model %d tokens" % (len(self.role), V))
        if not 0 <= int(end_id) < V or self.role[int(end_id)] != 0:
            raise ValueError("END (id %d) must be a neutral token of the rule" % int(end_id))
        if self.allowed_at_start(int(end_id), max_steps) < beam:
            raise ValueError("only %d tokens are allowed at step 0 under the rule: fewer than beam_size %d"
                             % (self.allowed_at_start(int(end_id), max_steps), beam))
        role = self.device_role(device)
        state = torch.empty(int(_lib.lib().lo_bracket_state_bytes(B, self.max_depth)), dtype=torch.uint8, device=device)
        br = _lib.BracketRule()
        br.role, br.n_kinds, br.max_depth, br.state = role.data_ptr(), max(self.n_kinds, 1), self.max_depth, state.data_ptr()
        return br, (role, state)


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
    return RaggedLayout(imgs, order, groups, counts, region_offsets(counts))


def encode_packed(encoder, lay, enc, device, encode=None):
    """Runs ``encoder`` once per shape group of ``lay`` and writes its output into the packed ``enc`` [regions, C] in decode
    order.  ``encode(encoder_out)``: optional, applied to each group's encoder output [n, H', W', C] before it is packed (the row
    encoder of ext.Img2SeqRowModel); its result has the same shape."""
    imgs, order, off = lay.imgs, lay.order, lay.off
    for j0, j1 in lay.groups:
        batch = torch.stack([imgs[order[j]] for j in range(j0, j1)]).to(device)
        e = encoder.forward_raw(batch if batch.dtype == torch.uint8 else batch.float(), need_grad=False)
        if encode is not None:
            e = encode(e)
        enc[off[j0]:off[j1]].copy_(e.reshape(off[j1] - off[j0], e.shape[3]))


def _prepare(model, img, rows_per_img, max_steps, encode=None):
    """Encoder output and the argument block of a decode of ``img``: a batch tensor, or a list of images of different sizes packed
    by ragged_layout.  ``encode``: as in encode_packed.  Returns (args, workspace, N, the RaggedLayout of a list or None)."""
    dec = model.decoder
    lay = None
    if isinstance(img, (list, tuple)):
        lay = ragged_layout(img, model.encoder.out_hw)
        N, R = len(lay.order), max(lay.counts)
        ws = decode_workspace(dec, N, R, rows_per_img, max_steps, lay.off)
        enc = ws["t"]["enc"]
        encode_packed(model.encoder, lay, enc, model.device, encode)
    else:
        enc = model.encoder.forward_raw(img.to(model.device).float(), need_grad=False)
        if encode is not None:
            enc = encode(enc)
        N, R = enc.shape[0], enc.shape[1] * enc.shape[2]
        enc = enc.view(N, R, enc.shape[3])
        ws = decode_workspace(dec, N, R, rows_per_img, max_steps)
    a = decode_args(dec, ws, enc, N, R, rows_per_img, max_steps, lay.off if lay is not None else None)
    return a, ws, N, lay


def decode_workspace(dec, N, R, rows_per_img, max_steps, off=None):
    """The workspace of a decode of N images x rows_per_img rows over at most R regions: for images of different sizes (``off``,
    their region offsets) the ragged one, whose packed encoder output ``ws["t"]["enc"]`` the caller fills; else the one of the
    shape, for an encoder output [N, R, C] of the caller's."""
    if off is not None:
        return dec.ragged_workspace(N * rows_per_img, max_steps, R, off[-1])
    return dec.workspace(N * rows_per_img, max_steps, R, need_grad=False)


def decode_args(dec, ws, enc, N, R, rows_per_img, max_steps, off=None):
    """The lo_decoder_args of a decode on ``ws`` (decode_workspace) once the encoder output ``enc`` is in place: every step runs
    all N * rows_per_img rows, the bf16 shadow refreshed, and with ``off`` the images' own region counts."""
    B = N * rows_per_img
    dec.store.refresh_shadow()
    for t in range(max_steps):
        ws["bt"][t] = B
    a = dec.fill_args(ws, enc, B, max_steps, R, has_dropout=False)
    a.rows_per_img = rows_per_img
    if off is not None:
        set_region_offsets(a, ws["reg_off_host"], ws["t"]["reg_off"], off)
    return a


def _inverse(order):
    inv = [0] * len(order)
    for j, i in enumerate(order):
        inv[i] = j
    return torch.tensor(inv, dtype=torch.int64)


def _greedy_entry(a, *args, br=None):
    if br is not None:
        return _lib.lib().lo_decoder_greedy_brackets(ctypes.byref(a), *args[:-1], ctypes.byref(br), args[-1])
    return _lib.lib().lo_decoder_greedy_hist(ctypes.byref(a), *args)


def _beam_entry(a, pen, *args, br=None):
    L = _lib.lib()
    if br is not None:
        return L.lo_decoder_beam_brackets(ctypes.byref(a), *args[:-1], ctypes.byref(pen) if pen is not None else None,
                                          ctypes.byref(br), args[-1])
    if pen is not None:
        return L.lo_decoder_beam_pen(ctypes.byref(a), *args[:-1], ctypes.byref(pen), args[-1])
    return L.lo_decoder_beam_div(ctypes.byref(a), *args)


def bracket_args(brackets, end_id, V, B, max_steps, device, beam=1):
    """(lo_bracket_rule or None, tensors to keep alive) of a decode under ``brackets`` (a BracketRule or None)."""
    if brackets is None:
        return None, None
    if not isinstance(brackets, BracketRule):
        raise TypeError("brackets must be a decode.BracketRule (got %s)" % type(brackets).__name__)
    return brackets.args(end_id, V, B, max_steps, device, beam)


def refuse_reference_finalize(brackets, finalize):
    """A bracket rule holds along hypothesis lineages only: 'reference' finalize (slot s of every step) is refused with it."""
    if brackets is not None and finalize != "backtrack":
        raise ValueError("a bracket rule needs finalize='backtrack': 'reference' returns slot s of every step, not a hypothesis's "
                         "lineage, so its sequences need not nest")


def greedy_decode(model, img, start_id, end_id, max_length_formula=150, return_attention=False, brackets=None, _encode=None,
                  _entry=_greedy_entry):
    """Returns token ids [N, steps] (CPU int64), steps as the reference's loop would have run.  ``return_attention=True`` also
    returns the attention weights of every step, [N, steps, R] fp32 on the CPU — what the reference collects in
    ``attention_mechanism.ctx_vector`` for visualize_attention.py (attention_mechanism.py:96-121).  For a list of images the ids
    are in input order and the attention weights are a list of [steps, R_i] tensors, R_i the image's own region count.

    ``brackets``: a BracketRule, under which every formula nests its brackets and closes them (lo_decoder_greedy_brackets).

    ``_encode`` (see encode_packed) and ``_entry(args, start_id, end_id, max_steps, tokens, finished, fin_hist, stream, br=None)``,
    the library call, let ext.greedy_decode run the two-layer decoder through this body."""
    max_steps = max_length_formula + 2
    with torch.no_grad():
        a, ws, N, lay = _prepare(model, img, 1, max_steps, _encode)
        finished = torch.zeros(N, dtype=torch.int32, device=model.device)
        br, keep = bracket_args(brackets, end_id, a.V, a.B, max_steps, model.device)
        kw = {"br": br} if br is not None else {}
        ids = run_greedy(lambda tokens, hist: _entry(a, int(start_id), int(end_id), max_steps, tokens, finished.data_ptr(), hist,
                                                     stream_ptr(), **kw),
                         N, max_steps, model.device).cpu()
        n = ids.shape[1]
        if lay is None:
            return (ids, ws["t"]["alphas"][:, :n].float().cpu()) if return_attention else ids
        inv = _inverse(lay.order)
        if return_attention:
            al = ws["t"]["alphas"].view(-1)[:N * max_steps * a.R].view(N, max_steps, a.R)[:, :n].cpu()
            return ids[inv], [al[j, :, :lay.counts[j]].clone() for j in inv.tolist()]
        return ids[inv]


def attention_maps(alphas, att_h, att_w):
    """visualize_attention.py:49-72 (getOutArray): an attention vector over the R = att_h * att_w regions as a grey image,
    region r at (r // att_w, r % att_w), value (1 - alpha) * 255 (dark = attended).  alphas [..., R] -> float [..., att_h, att_w]."""
    a = torch.as_tensor(alphas, dtype=torch.float32)
    if a.shape[-1] != att_h * att_w:
        raise ValueError("attention vector of %d regions does not match a %dx%d feature map" % (a.shape[-1], att_h, att_w))
    return ((1.0 - a) * 255.0).reshape(tuple(a.shape[:-1]) + (att_h, att_w))


def beam_decode(model, img, start_id, end_id, beam_size=5, max_length_formula=150, finalize="reference",
                div_gamma=1, div_prob=0, div_u=None, div_seed=None, return_attention=False, length_penalty=0.0,
                coverage_penalty=0.0, return_scores=False, brackets=None, _encode=None, _entry=_beam_entry):
    """Returns (ids [N, beam, steps], log_probs [N, beam]) on the CPU; hypothesis 0 is the one the reference scores
    (img2seq.py:210).  ``div_gamma`` / ``div_prob``: the diversity penalty of beam_search_decoder_cell.py:258-287 (off when
    gamma == 1 or prob == 0, as in configs/model.json:15-16); its Bernoulli draws come from the in-kernel Philox stream seeded
    by ``div_seed`` (default: torch's initial seed), or from ``div_u`` — uniforms [steps, N*beam, V] — when given (tests).  For a
    list of images, results are in input order and image i draws the rows [i*beam, (i+1)*beam) of ``div_u``.

    ``return_attention=True`` also returns the attention weights of every hypothesis, [N, beam, steps, R] fp32 on the CPU (a list
    of [beam, steps, R_i] for a list of images): under ``finalize='reference'`` the rows slot s computed at each step, what the
    reference's attention_mechanism.ctx_vector holds and visualize_attention.py draws for s = 0; under ``'backtrack'`` the
    attention under which each token of the hypothesis was chosen (the rows of a teacher-forced pass over its tokens).

    ``length_penalty`` (alpha) / ``coverage_penalty`` (beta): the penalties of GNMT (Wu et al. 2016) that lo_beam_penalty
    documents — the search ranks hypotheses by log_probs / ((5 + length) / 6) ** alpha + beta * sum_r ln(min(coverage_r, 1)), the
    coverage being the attention summed along the hypothesis.  Both default to 0, the reference's search.  The log-probs returned
    stay the raw sums; ``return_scores=True`` also returns the ranking scores [N, beam] (CPU), after the log-probs and before the
    attention weights.

    ``brackets``: a BracketRule (lo_decoder_beam_brackets): the search runs on the log-probs restricted to the tokens the rule
    allows, and every hypothesis nests its brackets and closes them.  It needs ``finalize='backtrack'`` (ValueError otherwise).

    ``_encode`` (see encode_packed) and ``_entry(args, penalty or None, start_id, end_id, max_steps, ids, parents, fin_hist, logp,
    div_gamma, div_prob, div_u, div_state, stream, br=None)``, the library call, let ext.beam_decode run the two-layer decoder
    through this body."""
    if finalize not in ("reference", "backtrack"):
        raise NotImplementedError("finalize must be 'reference' or 'backtrack'")
    refuse_reference_finalize(brackets, finalize)
    alpha, beta = penalty_weights(length_penalty, coverage_penalty)
    max_steps = max_length_formula + 2
    with torch.no_grad():
        a, ws, N, lay = _prepare(model, img, beam_size, max_steps, _encode)
        dev = model.device
        div_on = not (div_gamma == 1 or div_prob == 0)
        state = None
        if div_on and div_u is None:
            seed = torch.initial_seed() if div_seed is None else int(div_seed)
            state = torch.tensor([seed & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64, device=dev)

        pen = None
        if alpha != 0 or beta > 0 or return_scores:
            pen, pen_t = beam_penalty(alpha, beta, a.B, a.R, max_steps, beam_size, dev)
        br, keep = bracket_args(brackets, end_id, a.V, a.B, max_steps, dev, beam_size)
        kw = {"br": br} if br is not None else {}

        def call(ids, parents, hist, logp, u):
            return _entry(a, pen, int(start_id), int(end_id), max_steps, ids, parents, hist, logp, float(div_gamma), float(div_prob), u,
                          state.data_ptr() if state is not None else None, stream_ptr(), **kw)
        ids, parents, logp = run_beam(call, N, beam_size, max_steps, a.V, dev, div_u if div_on else None,
                                      lay.order if lay else None)
        scores = pen_t["scores"].cpu() if return_scores else None
        att = None
        if return_attention or finalize == "backtrack":
            alphas = ws["t"]["alphas"].view(-1)[:a.B * a.T * a.R].view(a.B, a.T, a.R) if return_attention else None
            ids, att = beam_hypotheses(ids, parents, finalize, a, alphas)
            ids, att = ids.cpu(), att.cpu() if att is not None else None
        else:
            ids = ids.cpu().permute(0, 2, 1).contiguous()     # [N, beam, time] like img2seq.py:239-241
        logp = logp.cpu()
        if lay is not None:
            inv = _inverse(lay.order)
            ids, logp = ids[inv], logp[inv]
            if scores is not None:
                scores = scores[inv]
            if att is not None:
                att = [att[j, :, :, :lay.counts[j]].clone() for j in inv.tolist()]
        return (ids, logp) + ((scores,) if return_scores else ()) + ((att,) if return_attention else ())


def sampling_settings(n_samples, temperature, top_k, top_p, V):
    """(n, tau, k, p) of a sampling decode as ints and floats; out-of-range values raise ValueError (lo_sample_args refuses the
    same, but only after the encoder has run)."""
    n, tau, k, p = int(n_samples), float(temperature), int(top_k), float(top_p)
    if not 1 <= n <= 16:
        raise ValueError("n_samples must lie in 1..16 (got %r)" % (n_samples,))
    if not (math.isfinite(tau) and tau > 0):
        raise ValueError("temperature must be finite and > 0 (got %r)" % (temperature,))
    if not 0 <= k <= V:
        raise ValueError("top_k must lie in 0..%d, 0 = off (got %r)" % (V, top_k))
    if not 0 < p <= 1:
        raise ValueError("top_p must lie in (0, 1], 1 = off (got %r)" % (top_p,))
    return n, tau, k, p


def sample_state(holder, seed, device):
    """The Philox {seed, call} device state of one sampling decode: a new one at call 0 for a given ``seed`` (the same seed repeats
    the draws), else ``holder``'s own, seeded from torch's initial seed on first use, whose call counter every decode advances."""
    if seed is not None:
        return torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64, device=device)
    if getattr(holder, "_sample_state", None) is None:
        holder._sample_state = torch.tensor([torch.initial_seed() & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64, device=device)
    return holder._sample_state


def run_sample(call, N, n, steps, tau, top_k, top_p, V, state, device, u=None, order=None):
    """Sampling decode of N images x n samples: ``call(args, tokens, fin_hist)`` runs the flavour's entry point with the
    lo_sample_args ``args`` and the device pointers of the outputs.  ``u``: None (Philox from ``state``) or injected uniforms
    [steps, N * n, V] in input order (``order``: the input index of each decode image).  Returns (ids [N, n, k], log-probs [N, n]) on
    the device in decode order, k the steps the reference's loop would have run."""
    s = _lib.SampleArgs()
    s.tau, s.top_k, s.top_p = tau, top_k, top_p
    logp = torch.zeros(N * n, dtype=torch.float32, device=device)
    s.logp = logp.data_ptr()
    if u is not None:
        u = torch.as_tensor(u, dtype=torch.float32).to(device).contiguous()
        if tuple(u.shape) != (steps, N * n, V):
            raise ValueError("u must be [steps, N * n_samples, V] = [%d, %d, %d]" % (steps, N * n, V))
        if order is not None:
            u = u.view(steps, N, n, V)[:, torch.tensor(order, device=device)].reshape(steps, N * n, V).contiguous()
        s.u = u.data_ptr()
    else:
        s.state = state.data_ptr()
    ids = run_greedy(lambda tokens, hist: call(s, tokens, hist), N * n, steps, device)
    return ids.reshape(N, n, -1), logp.view(N, n)


def _sample_entry(a, s, *args, br=None):
    if br is not None:
        return _lib.lib().lo_decoder_sample_brackets(ctypes.byref(a), ctypes.byref(s), *args[:-1], ctypes.byref(br), args[-1])
    return _lib.lib().lo_decoder_sample(ctypes.byref(a), ctypes.byref(s), *args)


def sample_decode(model, img, start_id, end_id, n_samples=8, temperature=1.0, top_k=0, top_p=1.0, max_length_formula=150,
                  seed=None, u=None, return_attention=False, brackets=None, _encode=None, _entry=_sample_entry):
    """Draws ``n_samples`` formulas per image (lo_decoder_sample): every step's token is a draw from softmax(logits /
    ``temperature``), restricted to the ``top_k`` most probable tokens (0: all) and to the smallest prefix of them, by probability,
    whose mass reaches ``top_p`` (1: all).  ``top_k = 1`` is greedy decode.  A sample ends at its first END (later positions hold
    END); the loop runs as long as greedy decode's, until every sample has ended.

    Returns (ids [N, n_samples, steps], log_probs [N, n_samples]) on the CPU; log_probs is each sample's log-likelihood under the
    model (temperature 1, no filter) through its first END, comparable with beam_decode's.  ``return_attention=True`` also returns
    the attention weights [N, n_samples, steps, R] fp32 (for a list of images, a list of [n_samples, steps, R_i]).  ``img``: a batch
    tensor or a list of images of different sizes, results in input order.

    The uniforms of the draws come from the in-kernel Philox stream: with ``seed``, a new stream at that seed (the same seed gives
    the same samples); without, the model's own stream, which every call advances.  ``u`` (tests): injected uniforms [steps, N *
    n_samples, V] in (0, 1), image i drawing the rows [i * n_samples, (i + 1) * n_samples).  ``mbr_select`` picks one sample per
    image from the result.

    ``brackets``: a BracketRule (lo_decoder_sample_brackets): the draws come from the model's distribution restricted to the
    tokens the rule allows (temperature, top_k and top_p act on it, and log_probs are restricted log-likelihoods), and every sample
    nests its brackets and closes them.

    ``_encode`` (see encode_packed) and ``_entry(args, sample_args, start_id, end_id, max_steps, tokens, finished, fin_hist,
    stream, br=None)``, the library call, let ext.sample_decode run the two-layer decoder through this body."""
    n, tau, k, p = sampling_settings(n_samples, temperature, top_k, top_p, model.decoder.vocab_size)
    max_steps = max_length_formula + 2
    with torch.no_grad():
        dev = model.device
        state = sample_state(model, seed, dev) if u is None else None
        a, ws, N, lay = _prepare(model, img, n, max_steps, _encode)
        finished = torch.zeros(a.B, dtype=torch.int32, device=dev)
        br, keep = bracket_args(brackets, end_id, a.V, a.B, max_steps, dev)
        kw = {"br": br} if br is not None else {}

        def call(s, tokens, hist):
            return _entry(a, s, int(start_id), int(end_id), max_steps, tokens, finished.data_ptr(), hist, stream_ptr(), **kw)
        ids, logp = run_sample(call, N, n, max_steps, tau, k, p, a.V, state, dev, u, lay.order if lay else None)
        ids, logp = ids.cpu(), logp.cpu()
        steps = ids.shape[2]
        att = None
        if return_attention:
            att = ws["t"]["alphas"].view(-1)[:a.B * max_steps * a.R].view(N, n, max_steps, a.R)[:, :, :steps].cpu()
        if lay is not None:
            inv = _inverse(lay.order)
            ids, logp = ids[inv], logp[inv]
            if att is not None:
                att = [att[j, :, :, :lay.counts[j]].clone() for j in inv.tolist()]
        return (ids, logp) + ((att,) if return_attention else ())


def mbr_select(ids, end_id):
    """Minimum-Bayes-risk choice among the samples of each image: ids [N, n, steps] (sample_decode) -> (choice [N] int64,
    agreement [N] fp32).  Every pair of samples of an image is scored with the edit-distance similarity of scst.rewards
    (layout="tf": 1 - lev / max length, each truncated at its first ``end_id``), all pairs of all images in one
    lo_scst_edit_reward launch; choice[i] is the sample with the highest mean similarity to the other samples (the lowest index
    among equals) and agreement[i] that mean, a confidence for the image.  With one sample: choice 0, agreement 1."""
    from . import scst
    ids = torch.as_tensor(ids)
    if ids.dim() != 3:
        raise ValueError("ids must be [N, n, steps] (got shape %s)" % (tuple(ids.shape),))
    N, n, _ = ids.shape
    if n == 1:
        return torch.zeros(N, dtype=torch.int64), torch.ones(N, dtype=torch.float32)
    i, j = torch.triu_indices(n, n, 1)                        # the similarity is symmetric: each unordered pair once
    dev = ids.device if ids.is_cuda else torch.device("cuda")
    x = ids.to(dev, torch.int64)
    r = scst.rewards(x[:, i].reshape(-1, x.shape[2]), x[:, j].reshape(-1, x.shape[2]), end_id, layout="tf")[0]
    r = r.view(N, -1).double().cpu()
    sim = torch.zeros(N, n, n, dtype=torch.float64)
    sim[:, i, j] = r
    sim[:, j, i] = r
    mean = sim.sum(dim=2) / (n - 1)
    choice = torch.argmax(mean, dim=1)                        # the first maximum
    return choice, mean.gather(1, choice.unsqueeze(1)).squeeze(1).float()


def truncate_end(list_of_ids, id_end):
    """model/evaluation/text.py:95-104."""
    out = []
    for seq in list_of_ids:
        seq = [int(t) for t in seq]
        out.append(seq[:seq.index(id_end)] if id_end in seq else seq)
    return out
