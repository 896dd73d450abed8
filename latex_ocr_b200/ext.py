"""EXTENSION beyond the reference — BASELINE.json configs[3]: "row-encoder biLSTM over CNN feature rows + 2-layer decoder,
160x640 images".  The reference contains neither (SURVEY.md §0: `model/decoder.py:16` only links the im2markup paper), so there
is no reference code to restate; semantics are defined HERE and checked against torch.nn.LSTM / autograd (oracle/ref_ext.py):

  RowEncoder        nn.LSTM(512, 256, bidirectional=True, batch_first=True) run over every ROW of the CNN feature map
                    ([N,H',W',512] -> [N,H',W',512], forward || backward halves), zero initial state; state_dict keys
                    ``lstm.weight_ih_l0 ... lstm.bias_hh_l0_reverse`` exactly like nn.LSTM.
  two-layer decoder the attention LSTM of DecoderWithAttention (seq2seq_torch.py:267-320) as layer 1; layer 2 =
                    nn.LSTMCell(D, D) over x_t = dropout(h1_t), zero initial state; logits_t = fc(h2_t).  Layer 2 does not feed
                    the attention, so it runs as one sequence LSTM between the time loop and the (hoisted) fc head
                    (``lo_decoder_args.phase`` 1 / 2).
  Img2SeqRowModel   EncoderCNN -> RowEncoder -> two-layer decoder, loss / regulariser / Adam exactly as Img2SeqModel.getLoss.

Both LSTMs run on ``lo_lstm_seq_forward/backward`` (csrc/lo_lstmseq.cuh): hoisted input projection, one recurrent GEMM + one cell
kernel per step, hand-derived backward with hoisted weight gradients.

Autograd: ``RowEncoder.forward`` and ``TwoLayerDecoder.forward`` (``Img2SeqRowModel.decoder2``) record a graph when grad mode is on
and an input or a parameter requires grad, so the whole extension trains through ``loss.backward()`` and ``torch.optim`` with any
loss of the predictions and alphas; the fused ``Img2SeqRowModel.train_step`` is unchanged.
"""
import ctypes
import itertools
import math

import torch
import torch.nn as nn

from . import _lib
from ._lib import check, ptr, stream_ptr
from .img2seq import Img2SeqModel
from .params import FlatStore, LRUCache, ParamHolder, grad_view, unbind_grads

# generation stamps of cached forward state: one counter for every cache, so a re-created (evicted) entry never repeats a stamp
_gen = itertools.count(1)


def _stamp(ent):
    ent["gen"] = next(_gen)
    return ent


def _live(snap):
    """snap: [(cache, key, entry, stamp)] taken at a forward.  True while no later forward rewrote or evicted any of them."""
    return all(c.get(k) is e and e["gen"] == g for c, k, e, g in snap)


def _snap(*pairs):
    return [(c, k, c[k], c[k]["gen"]) for c, k in pairs]


def _make_struct():
    with open(_lib.HEADER) as f:
        text = f.read()

    class LstmSeqArgs(ctypes.Structure):
        _fields_ = _lib._parse_struct(text, "lo_lstm_seq_args")

    return LstmSeqArgs


LstmSeqArgs = _make_struct()
_bound = False


def _bind():
    global _bound
    L = _lib.lib()
    if _bound:
        return L
    P = ctypes.POINTER(LstmSeqArgs)
    L.lo_sizeof_lstm_seq_args.restype = ctypes.c_int64
    if L.lo_sizeof_lstm_seq_args() != ctypes.sizeof(LstmSeqArgs):
        raise _lib.LatexOcrB200Error("lo_lstm_seq_args layout mismatch — rebuild")
    L.lo_lstm_seq_workspace_bytes.restype = ctypes.c_int64
    L.lo_lstm_seq_workspace_bytes.argtypes = [P]
    for name in ("lo_lstm_seq_forward", "lo_lstm_seq_backward"):
        fn = getattr(L, name)
        fn.argtypes = [P, ctypes.c_void_p]
        fn.restype = ctypes.c_int
    _bound = True
    return L


def _dt(precision):
    return _lib.LO_F32 if precision == "fp32" else _lib.LO_BF16


class _Direction:
    """One direction of one layer: argument block + workspace for a given (S, M) shape."""

    def __init__(self, store, prefix, suffix, I, H, precision, impl, reverse):
        self.store, self.I, self.H, self.precision, self.impl, self.reverse = store, I, H, precision, impl, reverse
        self.names = {k: "%s%s%s" % (prefix, k, suffix) for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")}
        self._ws = LRUCache()

    def args(self, S, M, stamp=False):
        """The argument block of shape (S, M); ``stamp``: this call writes the forward state (see _stamp)."""
        key = (S, M)
        ent = self._ws.get(key)
        S_ = self.store
        if ent is None:
            a = LstmSeqArgs()
            a.S, a.M, a.I, a.H = S, M, self.I, self.H
            a.dt = _dt(self.precision)
            a.impl = _lib.LO_IMPL_TC if (self.impl == "tc" and self.precision == "bf16") else _lib.LO_IMPL_SIMT
            a.reverse = 1 if self.reverse else 0
            nbytes = int(_bind().lo_lstm_seq_workspace_bytes(ctypes.byref(a)))
            ws = torch.zeros(nbytes, dtype=torch.uint8, device=S_.device)
            a.ws = ws.data_ptr()
            ent = self._ws[key] = {"a": a, "ws": ws}
        if stamp:
            _stamp(ent)
        a = ent["a"]
        n = self.names
        a.w_ih, a.w_hh = S_.w(n["weight_ih"]).data_ptr(), S_.w(n["weight_hh"]).data_ptr()
        a.b_ih, a.b_hh = S_.f32(n["bias_ih"]).data_ptr(), S_.f32(n["bias_hh"]).data_ptr()
        a.g_w_ih, a.g_w_hh = S_.g(n["weight_ih"]).data_ptr(), S_.g(n["weight_hh"]).data_ptr()
        a.g_b_ih, a.g_b_hh = S_.g(n["bias_ih"]).data_ptr(), S_.g(n["bias_hh"]).data_ptr()
        return a


def _lstm_specs(prefix, suffix, I, H):
    return [("%sweight_ih%s" % (prefix, suffix), (4 * H, I)), ("%sweight_hh%s" % (prefix, suffix), (4 * H, H)),
            ("%sbias_ih%s" % (prefix, suffix), (4 * H,)), ("%sbias_hh%s" % (prefix, suffix), (4 * H,))]


class RowEncoder(nn.Module):
    """Bidirectional LSTM over the rows of the CNN feature map (extension, see module docstring)."""

    def __init__(self, channels=512, hidden=256, device="cuda", precision="bf16", impl=None):
        super().__init__()
        self.C, self.H = channels, hidden
        self.precision = precision
        self.impl = impl if impl is not None else ("tc" if precision == "bf16" else "simt")
        self.tdtype = torch.float32 if precision == "fp32" else torch.bfloat16
        specs = _lstm_specs("lstm.", "_l0", channels, hidden) + _lstm_specs("lstm.", "_l0_reverse", channels, hidden)
        self.store = FlatStore(specs, device, bf16_shadow=(precision == "bf16"))
        self.lstm = ParamHolder()
        for name, _ in specs:
            self.lstm.bind(name.split(".", 1)[1], self.store, name)
        self.dirs = (_Direction(self.store, "lstm.", "_l0", channels, hidden, precision, self.impl, False),
                     _Direction(self.store, "lstm.", "_l0_reverse", channels, hidden, precision, self.impl, True))
        b = 1.0 / math.sqrt(hidden)                       # nn.LSTM.reset_parameters
        with torch.no_grad():
            for p_ in self.lstm.parameters():
                p_.uniform_(-b, b)
        self._out = LRUCache()
        self._shadow_fresh = False
        self._shadow_version = -1

    def _load_from_state_dict(self, *a, **k):
        super()._load_from_state_dict(*a, **k)
        self._shadow_fresh = False

    def sync_shadow(self):
        _sync_shadow(self)

    def forward_raw(self, feat):
        """feat: CUDA storage-dtype [N,H',W',C] -> storage-dtype [N,H',W',2*hidden] (a cached buffer)."""
        L = _bind()
        if not feat.is_cuda:
            raise _lib.LatexOcrB200Error("RowEncoder runs on CUDA tensors only (no CPU fallback)")
        feat = feat.contiguous().to(self.tdtype)
        N, Hh, Ww, C = feat.shape
        self.sync_shadow()
        ent = self._out.get((N, Hh, Ww))
        if ent is None:
            ent = self._out[(N, Hh, Ww)] = {"out": torch.empty(N, Hh, Ww, 2 * self.H, dtype=self.tdtype, device=feat.device),
                                           "dfeat": torch.empty(N, Hh, Ww, C, dtype=torch.float32, device=feat.device)}
        out = ent["out"]
        ent["feat"] = feat
        _stamp(ent)
        es = out.element_size()
        for d, dr in enumerate(self.dirs):
            a = dr.args(Ww, N * Hh, stamp=True)
            a.x, a.x_row, a.x_step = feat.data_ptr(), Ww * C, C
            a.hs = None
            a.hs_st = out.data_ptr() + d * self.H * es
            a.hs_row, a.hs_step = Ww * 2 * self.H, 2 * self.H
            check(L.lo_lstm_seq_forward(ctypes.byref(a), stream_ptr()))
        return out

    def backward_raw(self, shape, dout):
        """dout: fp32 [N,H',W',2*hidden] -> d feat fp32 [N,H',W',C]; parameter gradients land in self.store.grad."""
        L = _bind()
        N, Hh, Ww = shape
        ent = self._out[(N, Hh, Ww)]
        dfeat, feat = ent["dfeat"], ent["feat"]
        C = feat.shape[3]
        dout = dout.contiguous()
        for d, dr in enumerate(self.dirs):
            a = dr.args(Ww, N * Hh)
            a.x, a.x_row, a.x_step = feat.data_ptr(), Ww * C, C
            a.dhs = dout.data_ptr() + d * self.H * 4
            a.hs_row, a.hs_step = Ww * 2 * self.H, 2 * self.H
            a.dx, a.dx_row, a.dx_step, a.dx_accumulate = dfeat.data_ptr(), Ww * C, C, d
            check(L.lo_lstm_seq_backward(ctypes.byref(a), stream_ptr()))
        return dfeat

    def forward(self, feat):
        """feat [N,H',W',C] -> a fp32 [N,H',W',2*hidden] tensor.  With grad mode on and ``feat`` or a parameter requiring grad,
        an autograd graph is recorded whose backward runs ``backward_raw``; the output is the same either way."""
        params = list(self.parameters())
        if torch.is_grad_enabled() and (feat.requires_grad or any(p.requires_grad for p in params)):
            return _RowEncoderFunction.apply(self, feat, *params)
        with torch.no_grad():
            return self.forward_raw(feat).float()

    def _backward_impl(self, saved, dout, need_params):
        """(d feat in the caller's shape and dtype, [gradient or None per parameter]) of the forward ``saved`` describes."""
        N, Hh, Ww, C = saved["shape"]
        if not _live(saved["snap"]):
            raise _lib.LatexOcrB200Error(
                "RowEncoder backward: the saved forward state (N=%d, H'=%d, W'=%d) was overwritten by a later forward of the same "
                "shape (or of the same W' and N*H'); run backward before the next such forward" % (N, Hh, Ww))
        unbind_grads(self, self.store)           # the kernels overwrite store.grad
        dfeat = self.backward_raw((N, Hh, Ww), dout.float())
        dx = dfeat.to(saved["dtype"], copy=True)
        grads = [grad_view(self.store, p).clone() if need else None for p, need in zip(self.parameters(), need_params)]
        return dx, grads


def _sync_shadow(mod):
    # in-place edits of the parameters (torch.optim steps, load_state_dict, p.copy_) move the version counter that the views
    # share with store.master; the fused Adam writes the shadow itself and leaves the counter alone
    v = mod.store.master._version
    if not mod._shadow_fresh or v != mod._shadow_version:
        mod.store.sync_shadow()
        mod._shadow_fresh = True
        mod._shadow_version = v


class _RowEncoderFunction(torch.autograd.Function):
    """Autograd node of RowEncoder.forward: inputs (module, feat, *parameters), output the row encoding."""

    @staticmethod
    def forward(ctx, enc, feat, *params):
        out = enc.forward_raw(feat)
        N, Hh, Ww, C = feat.shape
        ctx.enc = enc
        ctx.saved = {"shape": (N, Hh, Ww, C), "dtype": feat.dtype,
                     "snap": _snap((enc._out, (N, Hh, Ww)), *((d._ws, (Ww, N * Hh)) for d in enc.dirs))}
        return out.clone() if out.dtype == torch.float32 else out.float()      # never the cached buffer itself

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dout):
        dx, grads = ctx.enc._backward_impl(ctx.saved, dout, ctx.needs_input_grad[2:])
        return (None, dx if ctx.needs_input_grad[1] else None) + tuple(grads)


class DecoderLayer2(nn.Module):
    """nn.LSTMCell(D, D) run over the whole sequence of dropout(h1_t) between the decoder's time loop and its fc head."""

    def __init__(self, D=512, device="cuda", precision="bf16", impl=None):
        super().__init__()
        self.D, self.precision = D, precision
        self.impl = impl if impl is not None else ("tc" if precision == "bf16" else "simt")
        self.tdtype = torch.float32 if precision == "fp32" else torch.bfloat16
        specs = _lstm_specs("cell.", "", D, D)
        self.store = FlatStore(specs, device, bf16_shadow=(precision == "bf16"))
        self.cell = ParamHolder()
        for name, _ in specs:
            self.cell.bind(name.split(".", 1)[1], self.store, name)
        self.dir = _Direction(self.store, "cell.", "", D, D, precision, self.impl, False)
        b = 1.0 / math.sqrt(D)
        with torch.no_grad():
            for p_ in self.cell.parameters():
                p_.uniform_(-b, b)
        self._shadow_fresh = False
        self._shadow_version = -1
        self._x = LRUCache()

    def _load_from_state_dict(self, *a, **k):
        super()._load_from_state_dict(*a, **k)
        self._shadow_fresh = False

    def sync_shadow(self):
        _sync_shadow(self)

    def saved_state(self, B, T):
        """What a later backward of the last forward of shape (B, T) needs to find unchanged (see ``state_live``)."""
        return (self._x[(B, T)], _snap((self.dir._ws, (T, B))))

    def state_live(self, state, B, T):
        return self._x.get((B, T)) is state[0] and _live(state[1])

    def forward_inplace(self, hd):
        """hd: fp32 [B,T,D] (dropout(h1), batch-major) — replaced IN PLACE by h2."""
        B, T, D = hd.shape
        self.sync_shadow()
        x = self._x.get((B, T))
        if x is None:
            x = self._x[(B, T)] = torch.empty(B, T, D, dtype=self.tdtype, device=hd.device)
        x.copy_(hd)                                        # layer input in storage dtype (plumbing cast)
        a = self.dir.args(T, B, stamp=True)
        a.x, a.x_row, a.x_step = x.data_ptr(), T * D, D
        a.hs, a.hs_st = hd.data_ptr(), None
        a.hs_row, a.hs_step = T * D, D
        check(_bind().lo_lstm_seq_forward(ctypes.byref(a), stream_ptr()))

    def backward_inplace(self, dhd):
        """dhd: fp32 [B,T,D] holding d loss / d h2 — replaced IN PLACE by d loss / d dropout(h1)."""
        B, T, D = dhd.shape
        a = self.dir.args(T, B)
        a.x, a.x_row, a.x_step = self._x[(B, T)].data_ptr(), T * D, D
        a.dhs = dhd.data_ptr()
        a.hs_row, a.hs_step = T * D, D
        a.dx, a.dx_row, a.dx_step, a.dx_accumulate = dhd.data_ptr(), T * D, D, 0      # d x is scattered after the loop has read dhs
        check(_bind().lo_lstm_seq_backward(ctypes.byref(a), stream_ptr()))


class _TwoLayerFunction(torch.autograd.Function):
    """Autograd node of TwoLayerDecoder.forward: inputs (module, side-output dict, encoder_out, captions, lengths, *parameters),
    differentiable outputs (predictions, alphas)."""

    @staticmethod
    def forward(ctx, dec2, rest, encoder_out, encoded_captions, caption_lengths, *params):
        preds, caps, decode_lengths, alphas, sort_ind, saved = dec2._forward_impl(encoder_out, encoded_captions, caption_lengths,
                                                                                  need_grad=True)
        rest["out"] = (caps, decode_lengths, sort_ind)
        ctx.dec2, ctx.saved = dec2, saved
        return preds, alphas

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dpreds, dalphas):
        dx, grads = ctx.dec2._backward_impl(ctx.saved, dpreds, dalphas, ctx.needs_input_grad[5:])
        return (None, None, dx if ctx.needs_input_grad[2] else None, None, None) + tuple(grads)


class TwoLayerDecoder(nn.Module):
    """The whole two-layer decoder as one module over an existing DecoderWithAttention (layer 1, attention, fc) and
    DecoderLayer2, whose parameters and state_dict entries stay where they are.  ``forward`` has DecoderWithAttention.forward's
    signature and return tuple; the phase protocol (time loop -> layer 2 over dropout(h1) -> fc head) stays inside."""

    def __init__(self, decoder, layer2):
        super().__init__()
        self.decoder, self.layer2 = decoder, layer2

    def _owned_params(self):
        return [(self.decoder, p) for p in self.decoder.parameters()] + [(self.layer2, p) for p in self.layer2.parameters()]

    def forward(self, encoder_out, encoded_captions, caption_lengths):
        """encoder_out [B,H',W',C] or [B,R,C]; returns (predictions [B,T,V], sorted captions, decode_lengths (list),
        alphas [B,T,R], sort_ind), rows sorted by length and outputs past a row's length zero.  With grad mode on and
        ``encoder_out`` or a parameter requiring grad, ``predictions`` and ``alphas`` are differentiable; the outputs are the
        same either way."""
        if not encoder_out.is_cuda:
            raise _lib.LatexOcrB200Error("TwoLayerDecoder runs on CUDA tensors only (no CPU fallback)")
        params = [p for _, p in self._owned_params()]
        if torch.is_grad_enabled() and (encoder_out.requires_grad or any(p.requires_grad for p in params)):
            rest = {}
            preds, alphas = _TwoLayerFunction.apply(self, rest, encoder_out, encoded_captions, caption_lengths, *params)
            caps, decode_lengths, sort_ind = rest["out"]
            return preds, caps, decode_lengths, alphas, sort_ind
        with torch.no_grad():
            return self._forward_impl(encoder_out, encoded_captions, caption_lengths, need_grad=False)[:5]

    def _forward_impl(self, encoder_out, encoded_captions, caption_lengths, need_grad):
        """The forward outputs, plus (need_grad) what the backward of this call needs."""
        dec, l2 = self.decoder, self.layer2
        B = encoder_out.size(0)
        C = encoder_out.size(-1)
        enc = encoder_out.reshape(B, -1, C)
        lens, sort_ind = caption_lengths.squeeze(1).sort(dim=0, descending=True)
        sort_ind_dev = sort_ind.to(enc.device)
        enc = enc[sort_ind_dev].contiguous().to(dec.tdtype)
        caps = encoded_captions.to(enc.device)[sort_ind_dev].contiguous()
        decode_lengths = (lens - 1).tolist()
        T = max(decode_lengths)
        mask = dec.make_dropout_mask(B, T)
        has_do = 0 if mask is None else (2 if isinstance(mask, str) else 1)
        # the Philox {seed, call} the dropout between the layers is drawn from; the backward regenerates the mask from this copy
        dstate = dec.dropout_state.clone() if need_grad and has_do == 2 else None
        ws = dec.run_forward(enc, caps, decode_lengths, with_loss=False, need_grad=need_grad, dropout_mask=mask, phase=1)
        l2.forward_inplace(ws["t"]["hd"])                  # hd: dropout(h1) -> h2
        dec.run_phase(ws, 2, backward=False, with_loss=False)
        if has_do == 2:
            dec.dropout_state[1] += 1        # forward-only call: no lo_decoder_backward to advance the Philox call counter
        preds = ws["t"]["logits"][:, :, :dec.vocab_size].clone()
        alphas = ws["t"]["alphas"].clone()
        if min(decode_lengths) < T:      # rows that stopped decoding keep zeros (layer 2 and fc ran over every row)
            act = torch.arange(T, device=enc.device)[None, :] < torch.tensor(decode_lengths, device=enc.device)[:, None]
            preds = preds * act[:, :, None]
            alphas = alphas * act[:, :, None]
        saved = None
        if need_grad:
            saved = {"ws": ws, "gen": ws["gen"], "l2": l2.saved_state(B, T), "enc": enc, "sort_ind": sort_ind_dev,
                     "shape": tuple(encoder_out.shape), "dtype": encoder_out.dtype, "has_do": has_do, "dstate": dstate}
        return preds, caps, decode_lengths, alphas, sort_ind_dev, saved

    def _backward_impl(self, saved, dpreds, dalphas, need_params):
        """Phase 2 (generic: d predictions -> dhd = d h2), layer 2's backward (dhd -> d dropout(h1)), phase 1 (generic, with
        d alphas): returns (d encoder_out in the caller's row order and shape, [gradient or None per parameter])."""
        dec, l2 = self.decoder, self.layer2
        ws, enc = saved["ws"], saved["enc"]
        B, R, _ = enc.shape
        T = ws["t"]["hd"].shape[1]
        if ws["gen"] != saved["gen"] or not l2.state_live(saved["l2"], B, T):
            raise _lib.LatexOcrB200Error(
                "TwoLayerDecoder backward: the saved forward state (B=%d, T=%d, R=%d) was overwritten by a later forward of the "
                "same shape; run backward before the next forward of that shape" % (B, T, R))
        V = dec.vocab_size
        dpred = dpreds.float().contiguous() if dpreds is not None else torch.zeros(B, T, V, device=enc.device)
        dal = dalphas.float().contiguous() if dalphas is not None else None
        unbind_grads(dec, dec.store)             # the kernels overwrite store.grad
        unbind_grads(l2, l2.store)
        a = dec.fill_args(ws, enc, B, T, R, saved["has_do"])
        dstate = None
        if saved["dstate"] is not None:
            dstate = saved["dstate"].clone()     # the phase-1 backward advances the counter it is given
            a.dropout_state = dstate.data_ptr()
        a.dpred_ext = dpred.data_ptr()           # the generic-mode flag, set for both phases
        a.dpred_stride = V
        dec.run_phase(ws, 2, backward=True)      # d predictions -> dhd = d h2 (+ fc gradients)
        l2.backward_inplace(ws["t"]["dhd"])      # -> d dropout(h1) (+ layer-2 gradients)
        if dal is not None:
            a.dalpha_ext = dal.data_ptr()
        dec.run_phase(ws, 1, backward=True)      # time loop of layer 1 + hoisted gradients -> denc
        denc = ws["t"]["denc"]
        dx = torch.empty_like(denc).index_copy_(0, saved["sort_ind"], denc)
        dx = dx.view(saved["shape"]).to(saved["dtype"])
        grads = [grad_view(mod.store, p).clone() if need else None for (mod, p), need in zip(self._owned_params(), need_params)]
        return dx, grads


class Img2SeqRowModel(Img2SeqModel):
    """EncoderCNN -> RowEncoder -> attention decoder with a second LSTM layer (extension).  Same trainer surface as
    Img2SeqModel (getLoss / train_step / train / ...); decoding (predict_batch) is not offered for this variant.  Through
    autograd: ``decoder2(row_encoder(encoder(img)), formula, lengths)`` -> any loss -> ``backward()``."""

    def getModel(self, model_name="Img2Seq"):
        super().getModel(model_name)
        self.row_encoder = RowEncoder(512, 256, device=self.device, precision=self.precision, impl=self.impl)
        self.layer2 = DecoderLayer2(512, device=self.device, precision=self.precision, impl=self.impl)
        self.decoder2 = TwoLayerDecoder(self.decoder, self.layer2)      # the two-layer decoder as one differentiable module
        return self

    def getOptimizer(self, lr_method="adam", lr=0.001):
        super().getOptimizer(lr_method, lr)
        self.row_encoder.store.ensure_adam(lr)
        self.layer2.store.ensure_adam(lr)

    def set_lr(self, lr):
        super().set_lr(lr)
        self.row_encoder.store.set_lr(lr)
        self.layer2.store.set_lr(lr)

    def predict_batch(self, *a, **k):
        raise NotImplementedError("the row-encoder / two-layer extension offers the training path only")

    def _keepalive(self):
        keep = super()._keepalive()
        keep += [list(self.row_encoder._out.values()), list(self.layer2._x.values()), list(self.layer2.dir._ws.values())]
        keep += [list(d._ws.values()) for d in self.row_encoder.dirs]
        return keep

    def _step_body(self, img, caps, decode_lengths, dropout_mask):
        N = img.shape[0]
        feat = self.encoder.forward_raw(img, need_grad=True)                       # [N,H',W',512] incl. the timing signal
        Hh, Ww = feat.shape[1], feat.shape[2]
        enc_out = self.row_encoder.forward_raw(feat)
        R = Hh * Ww
        dec = self.decoder
        enc_flat = enc_out.view(N, R, enc_out.shape[3])
        # phase 1: time loop of layer 1 (writes hd = dropout(h1)); layer 2 over the sequence; phase 2: fc head + loss
        ws = dec.run_forward(enc_flat, caps, decode_lengths, with_loss=True, need_grad=True, dropout_mask=dropout_mask, phase=1)
        self.layer2.forward_inplace(ws["t"]["hd"])
        dec.run_phase(ws, 2, backward=False)
        dec.run_phase(ws, 2, backward=True)                                         # fc backward -> dhd = d h2
        self.layer2.backward_inplace(ws["t"]["dhd"])
        dec.run_phase(ws, 1, backward=True)                                         # BPTT of layer 1 + hoisted gradients -> denc
        scale = 1.0
        if self.dist is not None:
            self.dist.reduce_async(dec.store.grad)
            self.dist.reduce_async(self.layer2.store.grad)
            scale = 1.0 / self.dist.world_size
        dfeat = self.row_encoder.backward_raw((N, Hh, Ww), ws["t"]["denc"].view(N, Hh, Ww, enc_out.shape[3]))
        if self.dist is not None:
            self.dist.reduce_async(self.row_encoder.store.grad)
            self.encoder.backward_raw(tuple(img.shape), dfeat, on_layer_grad=self.dist.layer_hook(self.encoder))
            self.dist.wait()
        else:
            self.encoder.backward_raw(tuple(img.shape), dfeat)
        self._adam(dec.store, scale, dec)
        self._adam(self.layer2.store, scale)
        self._adam(self.row_encoder.store, scale)
        self._adam(self.encoder.store, scale, self.encoder)
        self.layer2._shadow_fresh = self.row_encoder._shadow_fresh = True          # the fused Adam refreshed the bf16 shadows
        return ws["t"]["loss"]

    def state_dict(self):
        sd = super().state_dict()
        sd["row_encoder"], sd["layer2"] = self.row_encoder.state_dict(), self.layer2.state_dict()
        return sd

    def load_state_dict(self, sd):
        super().load_state_dict(sd)
        self.row_encoder.load_state_dict(sd["row_encoder"])
        self.layer2.load_state_dict(sd["layer2"])
