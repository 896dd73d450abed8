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

Decoding: ``greedy_decode`` / ``beam_decode`` below run CNN -> RowEncoder -> both decoder layers in one CUDA time loop
(``lo_decoder2_greedy`` / ``lo_decoder2_beam``, csrc/lo_decoder2.cuh) through the bodies of decode.greedy_decode / beam_decode.

Autograd: ``RowEncoder.forward`` and ``TwoLayerDecoder.forward`` (``Img2SeqRowModel.decoder2``) record a graph when grad mode is on
and an input or a parameter requires grad, so the whole extension trains through ``loss.backward()`` and ``torch.optim`` with any
loss of the predictions and alphas; the fused ``Img2SeqRowModel.train_step`` is unchanged.
"""
import ctypes
import math

import torch
import torch.nn as nn

from . import _lib, decode
from ._lib import LstmSeqArgs, check, dtype_code, impl_code, stream_ptr
from .img2seq import Img2SeqModel
from .kernel_module import kernel_forward, stamp
from .params import FlatStore, LRUCache, ParamHolder

_bind = _lib.lib          # the library with the lo_lstm_seq_* signatures set (lib() binds them along with the rest)


class _Direction:
    """One direction of one layer: argument block + workspace for a given (S, M) shape."""

    def __init__(self, store, prefix, suffix, I, H, precision, impl, reverse):
        self.store, self.I, self.H, self.precision, self.impl, self.reverse = store, I, H, precision, impl, reverse
        self.names = {k: "%s%s%s" % (prefix, k, suffix) for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")}
        self._ws = LRUCache()

    def args(self, S, M):
        """The argument block of shape (S, M)."""
        return self.entry(S, M)["a"]

    def entry(self, S, M):
        """The cache entry {"a": argument block, "ws": workspace} of shape (S, M), weight and gradient pointers refreshed."""
        key = (S, M)
        ent = self._ws.get(key)
        S_ = self.store
        if ent is None:
            a = LstmSeqArgs()
            a.S, a.M, a.I, a.H = S, M, self.I, self.H
            a.dt = dtype_code(self.precision)
            a.impl = impl_code(self.impl, self.precision)
            a.reverse = 1 if self.reverse else 0
            nbytes = int(_lib.lib().lo_lstm_seq_workspace_bytes(ctypes.byref(a)))
            ws = torch.zeros(nbytes, dtype=torch.uint8, device=S_.device)
            a.ws = ws.data_ptr()
            ent = self._ws[key] = {"a": a, "ws": ws}
        a = ent["a"]
        n = self.names
        a.w_ih, a.w_hh = S_.w(n["weight_ih"]).data_ptr(), S_.w(n["weight_hh"]).data_ptr()
        a.b_ih, a.b_hh = S_.f32(n["bias_ih"]).data_ptr(), S_.f32(n["bias_hh"]).data_ptr()
        a.g_w_ih, a.g_w_hh = S_.g(n["weight_ih"]).data_ptr(), S_.g(n["weight_hh"]).data_ptr()
        a.g_b_ih, a.g_b_hh = S_.g(n["bias_ih"]).data_ptr(), S_.g(n["bias_hh"]).data_ptr()
        return ent


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

    def forward_raw(self, feat):
        """feat: CUDA storage-dtype [N,H',W',C] -> storage-dtype [N,H',W',2*hidden] (a cached buffer)."""
        return self._forward(feat)[0]

    def _forward(self, feat):
        """forward_raw, plus the cache entries it wrote: (output entry, [entry of each direction])."""
        L = _lib.lib()
        if not feat.is_cuda:
            raise _lib.LatexOcrB200Error("RowEncoder runs on CUDA tensors only (no CPU fallback)")
        feat = feat.contiguous().to(self.tdtype)
        N, Hh, Ww, C = feat.shape
        self.store.refresh_shadow()
        ent = self._out.get((N, Hh, Ww))
        if ent is None:
            ent = self._out[(N, Hh, Ww)] = {"out": torch.empty(N, Hh, Ww, 2 * self.H, dtype=self.tdtype, device=feat.device),
                                           "dfeat": torch.empty(N, Hh, Ww, C, dtype=torch.float32, device=feat.device)}
        out = ent["out"]
        ent["feat"] = feat
        stamp(ent)
        es = out.element_size()
        dirs = []
        for d, dr in enumerate(self.dirs):
            de = stamp(dr.entry(Ww, N * Hh))
            a = de["a"]
            a.x, a.x_row, a.x_step = feat.data_ptr(), Ww * C, C
            a.hs = None
            a.hs_st = out.data_ptr() + d * self.H * es
            a.hs_row, a.hs_step = Ww * 2 * self.H, 2 * self.H
            check(L.lo_lstm_seq_forward(ctypes.byref(a), stream_ptr()))
            dirs.append(de)
        return out, (ent, dirs)

    def backward_raw(self, shape, dout, state=None):
        """dout: fp32 [N,H',W',2*hidden] -> d feat fp32 [N,H',W',C]; parameter gradients land in self.store.grad.  ``state``: the
        entries of the forward to differentiate, as _forward returns them (default: the cached ones of this shape)."""
        L = _lib.lib()
        N, Hh, Ww = shape
        ent, dirs = state if state is not None else (self._out[(N, Hh, Ww)], [dr.entry(Ww, N * Hh) for dr in self.dirs])
        dfeat, feat = ent["dfeat"], ent["feat"]
        C = feat.shape[3]
        dout = dout.contiguous()
        for d, de in enumerate(dirs):
            a = de["a"]
            a.x, a.x_row, a.x_step = feat.data_ptr(), Ww * C, C
            a.dhs = dout.data_ptr() + d * self.H * 4
            a.hs_row, a.hs_step = Ww * 2 * self.H, 2 * self.H
            a.dx, a.dx_row, a.dx_step, a.dx_accumulate = dfeat.data_ptr(), Ww * C, C, d
            check(L.lo_lstm_seq_backward(ctypes.byref(a), stream_ptr()))
        return dfeat

    def forward(self, feat):
        """feat [N,H',W',C] -> a fp32 [N,H',W',2*hidden] tensor.  With grad mode on and ``feat`` or a parameter requiring grad,
        an autograd graph is recorded whose backward runs ``backward_raw``; the output is the same either way."""
        return kernel_forward(self, (feat,), (feat,))[0][0]

    def _forward_impl(self, feat, need_grad):
        """((row encoding,), None, what the backward of this call needs or None)."""
        out, state = self._forward(feat)
        if not need_grad:
            return (out.float(),), None, None
        saved = {"entries": [state[0]] + state[1], "state": state, "shape": tuple(feat.shape), "dtype": feat.dtype}
        return (out.to(torch.float32, copy=True),), None, saved          # never the cached buffer itself

    def _backward_impl(self, saved, dout, need):
        """(d feat in the caller's shape and dtype,) of the forward ``saved`` describes."""
        N, Hh, Ww, _ = saved["shape"]
        dfeat = self.backward_raw((N, Hh, Ww), dout.float(), saved["state"])
        return (dfeat.to(saved["dtype"], copy=True),)


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
        self._x = LRUCache()
        self._scratch = LRUCache()

    def decode_layer(self, a):
        """The lo_decoder2_layer of a decode with the decoder args ``a``: the weights in storage dtype (bf16 shadow refreshed), the
        fp32 biases and a scratch buffer of lo_decoder2_scratch_bytes(a) bytes, cached per size.  The struct points at the store and
        the cache: it is valid until the next call that changes either."""
        self.store.refresh_shadow()
        nbytes = int(_lib.lib().lo_decoder2_scratch_bytes(ctypes.byref(a)))
        scratch = self._scratch.get(nbytes)
        if scratch is None:
            scratch = self._scratch[nbytes] = torch.empty(nbytes, dtype=torch.uint8, device=self.store.device)
        l2 = _lib.Decoder2Layer()
        l2.w_ih, l2.w_hh = self.store.w("cell.weight_ih").data_ptr(), self.store.w("cell.weight_hh").data_ptr()
        l2.b_ih, l2.b_hh = self.store.f32("cell.bias_ih").data_ptr(), self.store.f32("cell.bias_hh").data_ptr()
        l2.scratch = scratch.data_ptr()
        return l2

    def forward_inplace(self, hd):
        """hd: fp32 [B,T,D] (dropout(h1), batch-major) — replaced IN PLACE by h2.  Returns the cache entries it wrote (layer
        input, direction), which backward_inplace can be given."""
        B, T, D = hd.shape
        self.store.refresh_shadow()
        ent = self._x.get((B, T))
        if ent is None:
            ent = self._x[(B, T)] = {"x": torch.empty(B, T, D, dtype=self.tdtype, device=hd.device)}
        stamp(ent)
        ent["x"].copy_(hd)                                 # layer input in storage dtype (plumbing cast)
        de = stamp(self.dir.entry(T, B))
        a = de["a"]
        a.x, a.x_row, a.x_step = ent["x"].data_ptr(), T * D, D
        a.hs, a.hs_st = hd.data_ptr(), None
        a.hs_row, a.hs_step = T * D, D
        check(_lib.lib().lo_lstm_seq_forward(ctypes.byref(a), stream_ptr()))
        return ent, de

    def backward_inplace(self, dhd, state=None):
        """dhd: fp32 [B,T,D] holding d loss / d h2 — replaced IN PLACE by d loss / d dropout(h1).  ``state``: what forward_inplace
        returned (default: the cached entries of this shape)."""
        B, T, D = dhd.shape
        ent, de = state if state is not None else (self._x[(B, T)], self.dir.entry(T, B))
        a = de["a"]
        a.x, a.x_row, a.x_step = ent["x"].data_ptr(), T * D, D
        a.dhs = dhd.data_ptr()
        a.hs_row, a.hs_step = T * D, D
        a.dx, a.dx_row, a.dx_step, a.dx_accumulate = dhd.data_ptr(), T * D, D, 0      # d x is scattered after the loop has read dhs
        check(_lib.lib().lo_lstm_seq_backward(ctypes.byref(a), stream_ptr()))


def _refuse_sampling(p):
    if p:
        raise _lib.LatexOcrB200Error("scheduled sampling is not available with the second decoder layer: the layer sits between the "
                                     "LSTM cell and fc, so layer 1's time loop has no per-step prediction to feed back")


class TwoLayerDecoder(nn.Module):
    """The whole two-layer decoder as one module over an existing DecoderWithAttention (layer 1, attention, fc) and
    DecoderLayer2, whose parameters and state_dict entries stay where they are.  ``forward`` has DecoderWithAttention.forward's
    signature and return tuple; the phase protocol (time loop -> layer 2 over dropout(h1) -> fc head) stays inside."""

    def __init__(self, decoder, layer2):
        super().__init__()
        self.decoder, self.layer2 = decoder, layer2

    def forward(self, encoder_out, encoded_captions, caption_lengths, sampling_prob=0.0):
        """encoder_out [B,H',W',C] or [B,R,C]; returns (predictions [B,T,V], sorted captions, decode_lengths (list),
        alphas [B,T,R], sort_ind), rows sorted by length and outputs past a row's length zero.  With grad mode on and
        ``encoder_out`` or a parameter requiring grad, ``predictions`` and ``alphas`` are differentiable; the outputs are the
        same either way.  Scheduled sampling (``sampling_prob`` > 0) is refused: the second layer sits between the cell and fc,
        so the time loop of layer 1 has no per-step prediction to feed back."""
        _refuse_sampling(sampling_prob)
        (preds, alphas), (caps, decode_lengths, sort_ind) = kernel_forward(self, (encoder_out, encoded_captions, caption_lengths),
                                                                           (encoder_out,))
        return preds, caps, decode_lengths, alphas, sort_ind

    def _forward_impl(self, encoder_out, encoded_captions, caption_lengths, need_grad):
        """((predictions, alphas), (captions, decode_lengths, sort_ind), what the backward of this call needs or None)."""
        dec = self.decoder
        enc, caps, decode_lengths, sort_ind = dec._sorted_inputs(encoder_out, encoded_captions, caption_lengths)
        mask = dec.make_dropout_mask(enc.shape[0], max(decode_lengths))
        ws = dec.run_forward(enc, caps, decode_lengths, with_loss=False, need_grad=need_grad, dropout_mask=mask, phase=1)
        l2_state = self.layer2.forward_inplace(ws["t"]["hd"])      # hd: dropout(h1) -> h2
        dec.run_phase(ws, 2, backward=False, with_loss=False)
        # layer 2 and fc ran over every row: the outputs past a row's length are zeroed like the decoder's
        outs, side, saved = dec._outputs(ws, encoder_out, enc, caps, decode_lengths, sort_ind, mask, need_grad)
        if saved is not None:
            saved["entries"] += l2_state
            saved["l2"] = l2_state
        return outs, side, saved

    def _backward_impl(self, saved, dpreds, dalphas, need):
        """Phase 2 (generic: d predictions -> dhd = d h2), layer 2's backward (dhd -> d dropout(h1)), phase 1 (generic, with
        d alphas): returns (d encoder_out in the caller's row order and shape,)."""
        dec, ws = self.decoder, saved["ws"]
        a, keep = dec._generic_backward_args(saved, dpreds)       # d predictions: the generic-mode flag of both phases
        dal = dalphas.float().contiguous() if dalphas is not None else None
        dec.run_phase(ws, 2, backward=True)                        # d predictions -> dhd = d h2 (+ fc gradients)
        self.layer2.backward_inplace(ws["t"]["dhd"], saved["l2"])  # -> d dropout(h1) (+ layer-2 gradients)
        if dal is not None:
            a.dalpha_ext = dal.data_ptr()
        dec.run_phase(ws, 1, backward=True)                        # time loop of layer 1 + hoisted gradients -> denc
        return (dec._scatter_denc(saved),)


class Img2SeqRowModel(Img2SeqModel):
    """EncoderCNN -> RowEncoder -> attention decoder with a second LSTM layer (extension).  Same trainer surface as
    Img2SeqModel (getLoss / train_step / train / ...); predict_batch is not offered for this variant: it decodes through
    ext.greedy_decode / ext.beam_decode.  Through
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

    predict_images = predict_batch

    def set_sampling_prob(self, p):
        _refuse_sampling(float(p))

    def set_self_critical(self, temperature):
        if temperature:
            raise _lib.LatexOcrB200Error("self-critical training is not available with the second decoder layer: it samples inside "
                                         "layer 1's time loop, which has no per-step prediction (see scheduled sampling)")

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
        return ws["t"]["loss"]

    def state_dict(self):
        sd = super().state_dict()
        sd["row_encoder"], sd["layer2"] = self.row_encoder.state_dict(), self.layer2.state_dict()
        return sd

    def load_state_dict(self, sd):
        super().load_state_dict(sd)
        self.row_encoder.load_state_dict(sd["row_encoder"])
        self.layer2.load_state_dict(sd["layer2"])


# ------------------------------------------------------------------------------------------------ decoding
def _row_encode(model):
    """The row encoder as decode.encode_packed's ``encode``: CNN output [n,H',W',512] -> row encoding of the same shape."""
    return model.row_encoder.forward_raw


def greedy_decode(model, img, start_id, end_id, max_length_formula=150, return_attention=False, brackets=None):
    """Greedy decode of an Img2SeqRowModel: CNN -> row encoder -> two-layer decoder (layer 2 over h1_t, logits = fc(h2_t)) in one
    CUDA time loop (lo_decoder2_greedy).  Arguments, outputs and loop rules are those of decode.greedy_decode: ``img`` a batch
    tensor or a list of images of different sizes, the attention weights of layer 1 with ``return_attention``, a
    decode.BracketRule with ``brackets`` (lo_decoder2_greedy_brackets)."""
    def entry(a, *args, br=None):
        l2 = model.layer2.decode_layer(a)
        if br is not None:
            return _lib.lib().lo_decoder2_greedy_brackets(ctypes.byref(a), ctypes.byref(l2), *args[:-1], ctypes.byref(br), args[-1])
        return _lib.lib().lo_decoder2_greedy(ctypes.byref(a), ctypes.byref(l2), *args)
    return decode.greedy_decode(model, img, start_id, end_id, max_length_formula, return_attention, brackets,
                                _encode=_row_encode(model), _entry=entry)


def beam_decode(model, img, start_id, end_id, beam_size=5, **kw):
    """Beam search of an Img2SeqRowModel through the row encoder and the two-layer decoder (lo_decoder2_beam).  Keywords and return
    values are those of decode.beam_decode: max_length_formula, finalize, div_gamma / div_prob / div_u / div_seed,
    length_penalty / coverage_penalty, return_scores, return_attention, brackets (lo_decoder2_beam_brackets)."""
    def entry(a, pen, *args, br=None):
        l2 = model.layer2.decode_layer(a)
        p = ctypes.byref(pen) if pen is not None else None
        if br is not None:
            return _lib.lib().lo_decoder2_beam_brackets(ctypes.byref(a), ctypes.byref(l2), *args[:-1], p, ctypes.byref(br), args[-1])
        return _lib.lib().lo_decoder2_beam(ctypes.byref(a), ctypes.byref(l2), *args[:-1], p, args[-1])
    return decode.beam_decode(model, img, start_id, end_id, beam_size, _encode=_row_encode(model), _entry=entry, **kw)


def sample_decode(model, img, start_id, end_id, n_samples=8, **kw):
    """Sampling decode of an Img2SeqRowModel through the row encoder and the two-layer decoder (lo_decoder2_sample).  Keywords and
    return values are those of decode.sample_decode: temperature, top_k, top_p, max_length_formula, seed, u, return_attention,
    brackets (lo_decoder2_sample_brackets)."""
    def entry(a, s, *args, br=None):
        l2 = model.layer2.decode_layer(a)
        if br is not None:
            return _lib.lib().lo_decoder2_sample_brackets(ctypes.byref(a), ctypes.byref(l2), ctypes.byref(s), *args[:-1],
                                                          ctypes.byref(br), args[-1])
        return _lib.lib().lo_decoder2_sample(ctypes.byref(a), ctypes.byref(l2), ctypes.byref(s), *args)
    return decode.sample_decode(model, img, start_id, end_id, n_samples, _encode=_row_encode(model), _entry=entry, **kw)
