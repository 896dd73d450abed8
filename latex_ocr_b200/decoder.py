"""Attention / DecoderWithAttention — drop-ins for model/components/seq2seq_torch.py:160-320 on the
sm_90a kernels (lo_decoder.cu) through the C ABI.  Same constructors, forward signatures, return
tuples and ``state_dict`` keys:
  attention.{encoder_att,decoder_att,full_att}.{weight,bias}, embedding.weight,
  decode_step.{weight_ih,weight_hh,bias_ih,bias_hh}, init_h.*, init_c.*, f_beta.*, fc.*
"""
import ctypes
import math

import torch
import torch.nn as nn

from . import _lib, decode
from ._lib import check, dtype_code, impl_code, ptr, stream_ptr
from .kernel_module import kernel_forward, stamp
from .params import FlatStore, LRUCache, ParamHolder, grad_view


def decoder_specs(A, E, D, V, C):
    """Flat order: [decoder_att.W; f_beta.W; weight_hh] and their biases are contiguous so the per-step
    GEMM h -> (att2 | gate_pre | hh) and its weight gradient are single launches."""
    return [
        ("attention.encoder_att.weight", (A, C)), ("attention.encoder_att.bias", (A,)),
        ("attention.decoder_att.weight", (A, D)), ("f_beta.weight", (C, D)), ("decode_step.weight_hh", (4 * D, D)),
        ("attention.decoder_att.bias", (A,)), ("f_beta.bias", (C,)), ("decode_step.bias_hh", (4 * D,)),
        ("attention.full_att.weight", (1, A)), ("attention.full_att.bias", (1,)),
        ("embedding.weight", (V, E)),
        ("decode_step.weight_ih", (4 * D, E + C)), ("decode_step.bias_ih", (4 * D,)),
        ("init_h.weight", (D, C)), ("init_c.weight", (D, C)), ("init_h.bias", (D,)), ("init_c.bias", (D,)),
        ("fc.weight", (V, D)), ("fc.bias", (V,)),
    ]


class Attention(nn.Module):
    """seq2seq_torch.py:160-192.  Stand-alone use: forward(encoder_out[B,R,C], decoder_hidden[B,D])
    -> (context[B,C], alpha[B,R]).  Inside DecoderWithAttention the parameters are views into the
    decoder's flat store."""

    def __init__(self, encoder_dim, decoder_dim, attention_dim, device="cuda", precision="bf16", _store=None, impl=None):
        super().__init__()
        self.encoder_dim, self.decoder_dim, self.attention_dim = encoder_dim, decoder_dim, attention_dim
        self.precision = precision
        # GEMMs of the backward's two [B*R, A] x [A, C] products: wgmma in bf16 ("tc"), CUDA cores otherwise
        self.impl = impl if impl is not None else ("tc" if precision == "bf16" else "simt")
        self.tdtype = torch.float32 if precision == "fp32" else torch.bfloat16
        own = _store is None
        if own:
            specs = [("attention.encoder_att.weight", (attention_dim, encoder_dim)), ("attention.encoder_att.bias", (attention_dim,)),
                     ("attention.decoder_att.weight", (attention_dim, decoder_dim)), ("attention.decoder_att.bias", (attention_dim,)),
                     ("attention.full_att.weight", (1, attention_dim)), ("attention.full_att.bias", (1,))]
            _store = FlatStore(specs, device, bf16_shadow=(precision == "bf16"))
        self.store = _store
        for sub in ("encoder_att", "decoder_att", "full_att"):
            h = ParamHolder()
            h.bind("weight", _store, "attention.%s.weight" % sub)
            h.bind("bias", _store, "attention.%s.bias" % sub)
            setattr(self, sub, h)
        if own:
            with torch.no_grad():
                for sub, fan in (("encoder_att", encoder_dim), ("decoder_att", decoder_dim), ("full_att", attention_dim)):
                    b = 1.0 / math.sqrt(fan)
                    getattr(self, sub).weight.uniform_(-b, b)
                    getattr(self, sub).bias.uniform_(-b, b)
        self._work = None
        self._bwork = None

    def forward(self, encoder_out, decoder_hidden):
        """With grad mode on and ``encoder_out``, ``decoder_hidden`` or a parameter requiring grad, an autograd graph is
        recorded: ``context`` and ``alpha`` are differentiable, and their backward is lo_attention_step_backward.  The outputs
        are the same either way."""
        return kernel_forward(self, (encoder_out, decoder_hidden), (encoder_out, decoder_hidden))[0]

    def _forward_impl(self, encoder_out, decoder_hidden, need_grad):
        """((context, alpha), None, what the backward of this call needs or None).  att1 is computed per call, as the reference
        does (seq2seq_torch.py:186), and kept with att2 for the backward."""
        L = _lib.lib()
        with torch.no_grad():
            S, st, dt = self.store, stream_ptr(), dtype_code(self.precision)
            S.refresh_shadow()
            B, R, C = encoder_out.shape
            A, D = self.attention_dim, self.decoder_dim
            enc = encoder_out.contiguous().to(self.tdtype)
            att1 = torch.empty(B, R, A, dtype=self.tdtype, device=enc.device)
            check(L.lo_gemm(ptr(enc), dt, ptr(S.w("attention.encoder_att.weight")), dt, ptr(att1), dt, B * R, A, C,
                            C, 1, 1, C, A, 1, 0, 0, 0, ptr(S.f32("attention.encoder_att.bias")), 0, 0, _lib.LO_IMPL_SIMT, st))
            h = decoder_hidden.contiguous().float()
            att2 = torch.empty(B, A, dtype=torch.float32, device=enc.device)
            check(L.lo_gemm(ptr(h), _lib.LO_F32, ptr(S.w("attention.decoder_att.weight")), dt, ptr(att2), _lib.LO_F32, B, A, D,
                            D, 1, 1, D, A, 1, 0, 0, 0, ptr(S.f32("attention.decoder_att.bias")), 0, 0, _lib.LO_IMPL_SIMT, st))
            nbytes = L.lo_attention_workspace_bytes(B, C)
            if self._work is None or self._work.numel() < nbytes:
                self._work = torch.zeros(nbytes, dtype=torch.uint8, device=enc.device)
            alpha = torch.empty(B, R, dtype=torch.float32, device=enc.device)
            ctx = torch.empty(B, C, dtype=torch.float32, device=enc.device)
            check(L.lo_attention_forward(ptr(att1), ptr(enc), dt, ptr(att2), A, ptr(S.f32("attention.full_att.weight")),
                                         ptr(alpha), R, ptr(ctx), None, 0, None, B, R, A, C, ptr(self._work), st))
            saved = None
            if need_grad:
                # the caller's tensors are kept, not the storage-dtype / fp32 copies the kernels read: in a per-step loop the
                # enc[:bt] slices share one tensor, whereas a bf16 copy per call (57 MB at cfg #2) would double what the loop
                # holds; the backward redoes the same deterministic conversion (one cast per call)
                saved = {"tensors": (encoder_out, decoder_hidden, att1, att2, ctx, alpha),
                         "meta": {"version": S.master._version, "enc_shape": tuple(encoder_out.shape), "enc_dtype": encoder_out.dtype,
                                  "h_shape": tuple(decoder_hidden.shape), "h_dtype": decoder_hidden.dtype}}
            return (ctx, alpha), None, saved

    # the parameters in the order of lo_attention_step_backward's gradient arguments (and of self.parameters())
    _GRAD_NAMES = ("encoder_att.weight", "encoder_att.bias", "decoder_att.weight", "decoder_att.bias", "full_att.weight",
                   "full_att.bias")

    def _backward_impl(self, saved, dctx, dalpha, need):
        """lo_attention_step_backward: returns (d encoder_out or None, d decoder_hidden or None), each in the shape and dtype of
        what it is the gradient of; the parameter gradients ``need`` asks for land in ``store.grad``."""
        enc, h, att1, att2, ctx, alpha = saved["tensors"]
        meta = saved["meta"]
        S = self.store
        if S.master._version != meta["version"]:
            raise _lib.LatexOcrB200Error("Attention backward: a parameter was modified in place after the forward; run backward "
                                         "before the optimizer step")
        enc = enc.contiguous().to(self.tdtype)         # exactly what the forward's kernels read
        h = h.contiguous().float()
        B, R, C = enc.shape
        A, D = self.attention_dim, self.decoder_dim
        dev = enc.device
        f32 = torch.float32
        dctx = dctx.float().contiguous() if dctx is not None else torch.zeros(B, C, dtype=f32, device=dev)
        dal = dalpha.float().contiguous() if dalpha is not None else None
        named = dict(self.named_parameters())
        grads = [ptr(grad_view(S, named[n])) if nd else None for n, nd in zip(self._GRAD_NAMES, need[2:])]
        denc = torch.empty(B, R, C, dtype=f32, device=dev) if need[0] else None
        dh = torch.empty(B, D, dtype=f32, device=dev) if need[1] else None
        L = _lib.lib()
        dt = dtype_code(self.precision)
        nbytes = L.lo_attention_step_workspace_bytes(B, R, A, C, dt)
        if self._bwork is None or self._bwork.numel() < nbytes:
            self._bwork = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        check(L.lo_attention_step_backward(
            ptr(enc), ptr(att1), dt, ptr(h), ptr(att2), ptr(S.w("attention.encoder_att.weight")),
            ptr(S.w("attention.decoder_att.weight")), ptr(S.f32("attention.full_att.weight")), ptr(alpha), ptr(ctx), ptr(dctx),
            ptr(dal), ptr(denc), ptr(dh), *grads, None, None, None, B, R, A, C, D, impl_code(self.impl, self.precision),
            ptr(self._bwork), stream_ptr()))
        if denc is not None:
            denc = denc.view(meta["enc_shape"]).to(meta["enc_dtype"])
        if dh is not None:
            dh = dh.view(meta["h_shape"]).to(meta["h_dtype"])
        return denc, dh


class DecoderWithAttention(nn.Module):
    def __init__(self, attention_dim, embed_dim, decoder_dim, vocab_size, encoder_dim=512, dropout=0.5,
                 device="cuda", precision="bf16", impl=None):
        super().__init__()
        self.encoder_dim, self.attention_dim = encoder_dim, attention_dim
        self.embed_dim, self.decoder_dim, self.vocab_size = embed_dim, decoder_dim, vocab_size
        self.dropout_p = dropout
        self.precision = precision
        self.impl = impl if impl is not None else ("tc" if precision == "bf16" else "simt")
        self.alpha_c = 1.0                      # img2seq_torch.py:157
        self.tdtype = torch.float32 if precision == "fp32" else torch.bfloat16
        A, E, D, V, C = attention_dim, embed_dim, decoder_dim, vocab_size, encoder_dim
        self.store = FlatStore(decoder_specs(A, E, D, V, C), device, bf16_shadow=(precision == "bf16"))
        S = self.store
        self.attention = Attention(C, D, A, device, precision, _store=S, impl=self.impl)
        self.embedding = ParamHolder()
        self.embedding.bind("weight", S, "embedding.weight")
        self.dropout = nn.Dropout(p=dropout)    # kept for train()/eval() semantics and p
        self.decode_step = ParamHolder()
        for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
            self.decode_step.bind(n, S, "decode_step." + n)
        for n in ("init_h", "init_c", "f_beta", "fc"):
            h = ParamHolder()
            h.bind("weight", S, n + ".weight")
            h.bind("bias", S, n + ".bias")
            setattr(self, n, h)
        self.reset_parameters()
        self._ws = LRUCache()     # bounded: see params.LRUCache
        # in-kernel dropout (has_dropout=2): device {seed, call counter}; the counter is advanced by lo_decoder_backward, so
        # CUDA-graph replays draw a fresh mask every step
        self.dropout_state = torch.tensor([int(torch.initial_seed()) & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64, device=device)
        # scheduled sampling (forward(..., sampling_prob=p)): the device scalar p the kernels read, created on first use; the
        # tokens fed by the last forward ([B, T], sorted rows); injected coins [B, T] for parity tests (None: Philox)
        self._ss_prob = None
        self.last_fed_tokens = None
        self._ss_u = None
        # sampling with a temperature (forward(..., sampling_temperature=tau)): the device scalar tau, created on first use;
        # injected Gumbel uniforms [B, T, V] for parity tests (None: Philox)
        self._ss_temp = None
        self._ss_gu = None

    def seed_dropout(self, seed, call=0):
        self.dropout_state.copy_(torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, int(call)], dtype=torch.int64))

    def reset_parameters(self):
        A, E, D, V, C = self.attention_dim, self.embed_dim, self.decoder_dim, self.vocab_size, self.encoder_dim
        with torch.no_grad():
            def lin(h, fan):
                b = 1.0 / math.sqrt(fan)
                h.weight.uniform_(-b, b)
                h.bias.uniform_(-b, b)
            lin(self.attention.encoder_att, C)
            lin(self.attention.decoder_att, D)
            lin(self.attention.full_att, A)
            lin(self.init_h, C)
            lin(self.init_c, C)
            lin(self.f_beta, D)
            b = 1.0 / math.sqrt(D)
            for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                getattr(self.decode_step, n).uniform_(-b, b)
            self.embedding.weight.normal_(0, 1)
            lin(self.fc, D)
        self.init_weights()

    def init_weights(self):
        """seq2seq_torch.py:230-236."""
        with torch.no_grad():
            self.embedding.weight.uniform_(-0.1, 0.1)
            self.fc.bias.fill_(0)
            self.fc.weight.uniform_(-0.1, 0.1)

    def load_pretrained_embeddings(self, embeddings):
        """seq2seq_torch.py:238-244 (copies into the flat store instead of re-pointing the Parameter)."""
        with torch.no_grad():
            self.embedding.weight.copy_(embeddings)

    def fine_tune_embeddings(self, fine_tune=True):
        """seq2seq_torch.py:246-253."""
        for p in self.embedding.parameters():
            p.requires_grad = fine_tune

    # ---------------------------------------------------------------------------------------------
    def workspace(self, B, T, R, need_grad, key=None, att1_rows=None):
        """``att1_rows``: att1 as [att1_rows, A] (the packed layout of ragged_workspace) instead of [B, R, A]."""
        key = (B, T, R) if key is None else key
        ws = self._ws.get(key)
        dev = self.store.device
        A, E, D, V, C = self.attention_dim, self.embed_dim, self.decoder_dim, self.vocab_size, self.encoder_dim
        O1, G = A + C + 4 * D, 4 * D
        f32 = torch.float32

        def z(*shape, dtype=f32):
            return torch.zeros(*shape, dtype=dtype, device=dev)

        if ws is None:
            ws = {"need_grad": False}
            t = ws["t"] = {}
            t["caps"] = z(B, T + 1, dtype=torch.int64)
            t["att1"] = z(B, R, A, dtype=self.tdtype) if att1_rows is None else z(att1_rows, A, dtype=self.tdtype)
            t["ptab"] = z(V, G)
            t["mean"] = z(B, C)
            t["hall"] = z(T + 1, B, D)
            t["call"] = z(T + 1, B, D)
            t["out1"] = z(T, B, O1)
            t["alphas"] = z(B, T, R)
            t["ctx"] = z(T, B, C)
            t["gctx"] = z(T, B, C)
            t["gates"] = z(T, B, G)
            t["gtmp"] = z(B, G)
            t["hd"] = z(B, T, D)
            ws["ldl"] = (V + 63) // 64 * 64
            t["logits"] = z(B, T, ws["ldl"])
            t["row_loss"] = z(B * T + B * R)
            t["loss"] = z(4)
            t["sreg"] = z(B, max(T, 2))
            t["work"] = z(int(_lib.lib().lo_decoder_workspace_bytes(B, max(A, C))), dtype=torch.uint8)
            t["dropout_mask"] = None             # [B,T,D] allocated on first use of an injected mask
            ws["bt"] = (ctypes.c_int32 * T)(*([B] * T))
            self._ws[key] = ws
        stamp(ws)              # every caller overwrites the forward state: a pending autograd backward of it must refuse to run
        if need_grad and not ws["need_grad"]:
            t = ws["t"]
            t["wbwd1"] = z(C + D, G, dtype=self.tdtype)
            t["wbwd2"] = z(D, A + C, dtype=self.tdtype)
            t["dlogits"] = z(B, T, ws["ldl"])
            t["dhd"] = z(B, T, D)
            t["dreg"] = z(B, R)
            t["dcat"] = z(T, B, O1)
            t["dxh"] = z(B, C + D)
            t["dc"] = z(2, B, D)
            t["dctx"] = z(T, B, C)
            t["de"] = z(B, T, R)
            t["dptab"] = z(V, G)
            t["datt1"] = z(B, R, A, dtype=self.tdtype)
            t["denc"] = z(B, R, C)
            t["dinit"] = z(B, 2 * D)
            t["dmean"] = z(B, max(A, C))
            # ReLU mask bits of every step (forward attention kernel -> backward attention kernel), 1 bit per att1 element
            t["att_mask"] = torch.empty(T, B, (R + 1) // 2 * 2, A // 8, dtype=torch.uint8, device=dev)      # rows padded to an even count
            ws["need_grad"] = True
        return ws

    def ragged_workspace(self, B, T, R, n_regions):
        """Decode workspace for images of different sizes (lo_decoder_args.reg_off): the packed encoder output ``t["enc"]``
        [regions, C], att1 [regions, A] and every per-row buffer, sized by capacity (rows B, steps T, largest region count R,
        total regions; decode.ragged_cache)."""
        def build(B, T, R, n_regions):
            ws = self.workspace(B, T, R, False, key="ragged", att1_rows=n_regions)
            dev = self.store.device
            ws["t"]["enc"] = torch.zeros(n_regions, self.encoder_dim, dtype=self.tdtype, device=dev)
            ws["t"]["reg_off"] = torch.zeros(B + 1, dtype=torch.int32, device=dev)
            ws["reg_off_host"] = (ctypes.c_int32 * (B + 1))()
            self.fill_args(ws, ws["t"]["enc"], B, T, R, has_dropout=False)        # sizes bfwork (wgmma staging) by capacity
            return ws
        return decode.ragged_cache(self._ws, (B, T, R, n_regions), build)

    def _fed_buffer(self, ws):
        """[B, T] int64 tokens fed by a scheduled-sampling forward (allocated on first use of the mode for this shape)."""
        t = ws["t"]
        if t.get("fed") is None:
            t["fed"] = torch.zeros(t["hd"].shape[0], t["hd"].shape[1], dtype=torch.int64, device=self.store.device)
        return t["fed"]

    def _ws_for(self, B, T, R):
        """The cached workspace of an exact shape (tests / bench probes)."""
        return self._ws[(B, T, R)]

    def fill_args(self, ws, enc, B, T, R, has_dropout, dalpha_ext=None, ss_prob=None, ss_temp=None):
        S, t = self.store, ws["t"]
        a = _lib.DecoderArgs()
        a.B, a.T, a.R = B, T, R
        a.C, a.A, a.D, a.E, a.V = self.encoder_dim, self.attention_dim, self.decoder_dim, self.embed_dim, self.vocab_size
        a.dt = dtype_code(self.precision)
        a.impl = impl_code(self.impl, self.precision)
        a.has_dropout = int(has_dropout)           # 0 eval, 1 injected mask, 2 in-kernel Philox
        a.dropout_state = self.dropout_state.data_ptr()
        a.dropout_p = float(self.dropout_p)
        a.ldl = ws["ldl"]
        a.alpha_c = float(self.alpha_c)
        a.bt_host = ctypes.cast(ws["bt"], ctypes.c_void_p)
        a.caps = t["caps"].data_ptr()
        a.caps_stride = t["caps"].stride(0)
        a.enc = enc.data_ptr()

        def W(name):
            return S.w(name).data_ptr()

        def F(name):
            return S.f32(name).data_ptr()

        def Gd(name):
            return S.g(name).data_ptr()

        a.w_enc_att, a.b_enc_att = W("attention.encoder_att.weight"), F("attention.encoder_att.bias")
        a.wcat1, a.bcat1 = W("attention.decoder_att.weight"), F("attention.decoder_att.bias")
        a.w_full = F("attention.full_att.weight")
        a.emb = W("embedding.weight")
        a.w_ih, a.b_ih = W("decode_step.weight_ih"), F("decode_step.bias_ih")
        a.w_init, a.b_init = W("init_h.weight"), F("init_h.bias")
        a.w_fc, a.b_fc = W("fc.weight"), F("fc.bias")
        for k in ("att1", "ptab", "mean", "hall", "call", "out1", "alphas", "ctx", "gctx", "gates", "gtmp", "hd", "logits",
                  "row_loss", "loss", "sreg", "work"):
            setattr(a, k, t[k].data_ptr())
        if t.get("dropout_mask") is not None:
            a.dropout_mask = t["dropout_mask"].data_ptr()
        if ws["need_grad"]:
            for k in ("wbwd1", "wbwd2", "dlogits", "dhd", "dreg", "dcat", "dxh", "dc", "dctx", "de", "dptab", "datt1", "denc",
                      "dinit", "dmean", "att_mask"):
                setattr(a, k, t[k].data_ptr())
            a.g_w_enc_att, a.g_b_enc_att = Gd("attention.encoder_att.weight"), Gd("attention.encoder_att.bias")
            a.g_wcat1, a.g_bcat1 = Gd("attention.decoder_att.weight"), Gd("attention.decoder_att.bias")
            a.g_w_full, a.g_b_full = Gd("attention.full_att.weight"), Gd("attention.full_att.bias")
            a.g_emb = Gd("embedding.weight")
            a.g_w_ih, a.g_b_ih = Gd("decode_step.weight_ih"), Gd("decode_step.bias_ih")
            a.g_w_init, a.g_b_init = Gd("init_h.weight"), Gd("init_h.bias")
            a.g_w_fc, a.g_b_fc = Gd("fc.weight"), Gd("fc.bias")
        if dalpha_ext is not None:
            a.dalpha_ext = dalpha_ext.data_ptr()
        if ss_prob is not None:                    # scheduled sampling: device p, the fed-token record, injected coins if any
            a.ss_prob = ss_prob.data_ptr()
            a.fed = self._fed_buffer(ws).data_ptr()
            if self._ss_u is not None:
                a.ss_u = self._ss_u.data_ptr()
            if ss_temp is not None:                # a draw from softmax(logits / tau) instead of the argmax
                a.ss_temp = ss_temp.data_ptr()
                if self._ss_gu is not None:
                    a.ss_gu = self._ss_gu.data_ptr()
        if a.impl == _lib.LO_IMPL_TC:
            if "bfwork" not in t:
                t["bfwork"] = torch.zeros(int(_lib.lib().lo_decoder_bfwork_bytes(ctypes.byref(a))), dtype=torch.uint8, device=S.device)
            a.bfwork = t["bfwork"].data_ptr()
        ws["args"] = a
        return a

    def set_lengths(self, ws, decode_lengths, B, T):
        """bt[t] = number of rows still decoding at step t (seq2seq_torch.py:308)."""
        for t in range(T):
            ws["bt"][t] = sum(1 for l in decode_lengths if l > t)

    def init_hidden_state(self, encoder_out):
        """seq2seq_torch.py:255-265 (stand-alone; the fused path computes it inside lo_decoder_forward)."""
        L = _lib.lib()
        with torch.no_grad():
            S, st, dt = self.store, stream_ptr(), dtype_code(self.precision)
            S.refresh_shadow()
            m = encoder_out.float().mean(dim=1).contiguous()      # plumbing; the hot path uses mean_rows_kernel
            B, C, D = m.shape[0], self.encoder_dim, self.decoder_dim
            hc = torch.empty(2, B, D, dtype=torch.float32, device=m.device)
            for i, n in enumerate(("init_h", "init_c")):
                check(L.lo_gemm(ptr(m), _lib.LO_F32, ptr(S.w(n + ".weight")), dt, ptr(hc[i]), _lib.LO_F32, B, D, C, C, 1, 1, C, D,
                                1, 0, 0, 0, ptr(S.f32(n + ".bias")), 0, 0, _lib.LO_IMPL_SIMT, st))
            return hc[0], hc[1]

    def run_phase(self, ws, phase, backward, with_loss=True):
        """Extension hook (a second layer between the cell and fc, latex_ocr_b200/ext.py): re-enter the C entry points with
        ``lo_decoder_args.phase`` = 1 (time loop only) or 2 (fc head + loss only) on the argument block of run_forward.
        ``with_loss=False``: the phase-2 forward writes the logits only (the autograd path)."""
        a = ws["args"]
        a.phase = int(phase)
        try:
            L = _lib.lib()
            if backward:
                check(L.lo_decoder_backward(ctypes.byref(a), stream_ptr()))
            else:
                check(L.lo_decoder_forward(ctypes.byref(a), 1 if with_loss else 0, stream_ptr()))
        finally:
            a.phase = 0

    def run_forward(self, enc_flat, caps_sorted, decode_lengths, with_loss, need_grad, dropout_mask=None, phase=0, ss_prob=None,
                    ss_temp=None, key=None):
        """enc_flat: storage-dtype CUDA [B,R,C] (sorted rows); caps_sorted: CUDA int64 [B,T+1].
        dropout_mask: None (no dropout), a [B,T,D] tensor of multipliers (injected, parity tests) or the string "philox"
        (mask drawn inside the kernels).  ss_prob: None (teacher forcing) or a CUDA float32 scalar p: scheduled sampling, the
        tokens fed land in ``ws["t"]["fed"]`` (the same argument block serves the backward, run_backward).  ss_temp: None or a CUDA
        float32 scalar tau: a step that samples feeds a draw from softmax(logits / tau).  key: the workspace cache key (default
        (B, T, R)), so that two forwards of one shape keep separate state."""
        L = _lib.lib()
        B, R, _ = enc_flat.shape
        T = max(decode_lengths)
        ws = self.workspace(B, T, R, need_grad, key=key)
        self.store.refresh_shadow()
        ws["t"]["caps"].copy_(caps_sorted[:, :T + 1])
        self.set_lengths(ws, decode_lengths, B, T)
        has_do = 0 if dropout_mask is None else (2 if isinstance(dropout_mask, str) else 1)
        if has_do == 1:
            if ws["t"].get("dropout_mask") is None:
                ws["t"]["dropout_mask"] = torch.zeros(B, T, self.decoder_dim, dtype=torch.float32, device=self.store.device)
                ws.pop("args", None)
            ws["t"]["dropout_mask"].copy_(dropout_mask)
        a = self.fill_args(ws, enc_flat, B, T, R, has_do, ss_prob=ss_prob, ss_temp=ss_temp)
        a.phase = int(phase)
        try:
            check(L.lo_decoder_forward(ctypes.byref(a), 1 if with_loss else 0, stream_ptr()))
        finally:
            a.phase = 0
        return ws

    def run_backward(self, ws):
        check(_lib.lib().lo_decoder_backward(ctypes.byref(ws["args"]), stream_ptr()))

    def make_dropout_mask(self, B, T, materialize=False):
        """Dropout of h before fc (seq2seq_torch.py:316).  Training mode: "philox" = the inverted-dropout multipliers are drawn
        inside the LSTM kernels (csrc/lo_common.cuh:philox_dropout_mult) and redrawn in the backward — no mask tensor, no torch
        RNG launch; ``materialize=True`` returns the [B,T,D] tensor of torch-drawn multipliers instead (the injected-mask path
        the parity tests use)."""
        p = self.dropout_p
        if not self.training or p <= 0.0:
            return None
        if not materialize:
            return "philox"
        keep = torch.rand(B, T, self.decoder_dim, device=self.store.device) >= p
        return keep.float() / (1.0 - p)

    def forward(self, encoder_out, encoded_captions, caption_lengths, sampling_prob=0.0, sampling_temperature=0.0):
        """Reference signature and return tuple (seq2seq_torch.py:267-320): (predictions[B,maxT,V],
        sorted captions, decode_lengths(list), alphas[B,maxT,R], sort_ind).  With grad mode on and ``encoder_out`` or a
        parameter requiring grad, an autograd graph is recorded: ``predictions`` and ``alphas`` are differentiable (any loss of
        them), and their backward runs lo_decoder_backward in its generic mode.  The outputs are the same either way.

        ``sampling_prob`` = p > 0: scheduled sampling (Bengio et al. 2015) inside the CUDA time loop.  Step t >= 1 of a row feeds
        the argmax of the row's returned prediction of step t-1 (lowest index on ties) where a coin u ~ U[0,1) is below p, the
        teacher token ``captions[b][t]`` otherwise; step 0 feeds ``captions[b][0]``.  The coins come from Philox keyed by the
        dropout seed (one call counter per forward, also in eval mode; ``seed_dropout`` reproduces them).  Targets of a loss stay
        ``captions[:, 1:]``; the choice is not differentiated: the backward is teacher forcing on the tokens fed, which
        ``last_fed_tokens`` holds ([B, T] in sorted-row order, the teacher token past a row's length).  p = 0 runs the teacher-forced
        path unchanged (``last_fed_tokens`` is then ``captions[:, :T]``).

        ``sampling_temperature`` = tau > 0 (with p > 0): a step that samples feeds a draw from softmax(prediction / tau) (Gumbel-max,
        the uniforms from the same Philox call: ``philox.gumbel_uniforms``) instead of the argmax.  With p = 1 the call samples a
        whole sequence, and the outputs stay differentiable: log pi(sample) is a function of ``predictions`` and the tokens in
        ``last_fed_tokens``, so a policy-gradient loss (self-critical training, ``scst``) works through ``loss.backward()``.  0 (the
        default) is the argmax path, bit for bit."""
        (preds, alphas), (caps, decode_lengths, sort_ind) = kernel_forward(
            self, (encoder_out, encoded_captions, caption_lengths, float(sampling_prob), float(sampling_temperature or 0.0)),
            (encoder_out,))
        return preds, caps, decode_lengths, alphas, sort_ind

    def _forward_impl(self, encoder_out, encoded_captions, caption_lengths, sampling_prob=0.0, sampling_temperature=0.0,
                      need_grad=False):
        """((predictions, alphas), (captions, decode_lengths, sort_ind), what the backward of this call needs or None)."""
        if not 0.0 <= sampling_prob <= 1.0:
            raise ValueError("sampling_prob must lie in [0, 1] (got %r)" % (sampling_prob,))
        if not (sampling_temperature >= 0.0 and math.isfinite(sampling_temperature)):
            raise ValueError("sampling_temperature must be a finite tau >= 0 (got %r)" % (sampling_temperature,))
        if sampling_temperature > 0.0 and sampling_prob == 0.0:
            raise ValueError("sampling_temperature needs sampling_prob > 0: it sets how the fed tokens are drawn")
        enc, caps, decode_lengths, sort_ind = self._sorted_inputs(encoder_out, encoded_captions, caption_lengths)
        T = max(decode_lengths)
        mask = self.make_dropout_mask(enc.shape[0], T)
        ss = None
        if sampling_prob > 0.0:
            if self._ss_prob is None:
                self._ss_prob = torch.zeros((), dtype=torch.float32, device=self.store.device)
            ss = self._ss_prob
            ss.fill_(sampling_prob)
        tau = None
        if sampling_temperature > 0.0:
            if self._ss_temp is None:
                self._ss_temp = torch.zeros((), dtype=torch.float32, device=self.store.device)
            tau = self._ss_temp
            tau.fill_(sampling_temperature)
        ws = self.run_forward(enc, caps, decode_lengths, with_loss=False, need_grad=need_grad, dropout_mask=mask, ss_prob=ss,
                              ss_temp=tau)
        self.last_fed_tokens = ws["t"]["fed"].clone() if ss is not None else caps[:, :T]
        return self._outputs(ws, encoder_out, enc, caps, decode_lengths, sort_ind, mask, need_grad, sampling=ss is not None)

    def _backward_impl(self, saved, dpreds, dalphas, need):
        """lo_decoder_backward in its generic mode: returns (d encoder_out in the caller's row order and shape,)."""
        a, keep = self._generic_backward_args(saved, dpreds)
        dal = dalphas.float().contiguous() if dalphas is not None else None
        if dal is not None:
            a.dalpha_ext = dal.data_ptr()
        check(_lib.lib().lo_decoder_backward(ctypes.byref(a), stream_ptr()))
        return (self._scatter_denc(saved),)

    # shared with ext.TwoLayerDecoder, which runs its second layer between phase 1 (time loop) and phase 2 (fc head)
    def _sorted_inputs(self, encoder_out, encoded_captions, caption_lengths):
        """seq2seq_torch.py:284-298: (encoder_out as [B,R,C] in storage dtype, captions, decode_lengths, sort_ind), rows sorted by
        decreasing caption length."""
        B = encoder_out.size(0)
        C = encoder_out.size(-1)
        enc = encoder_out.reshape(B, -1, C)
        lens, sort_ind = caption_lengths.squeeze(1).sort(dim=0, descending=True)     # :286
        sort_ind = sort_ind.to(enc.device)
        enc = enc[sort_ind].contiguous().to(self.tdtype)
        caps = encoded_captions.to(enc.device)[sort_ind].contiguous()
        return enc, caps, (lens - 1).tolist(), sort_ind                             # :298

    def _outputs(self, ws, encoder_out, enc, caps, decode_lengths, sort_ind, mask, need_grad, sampling=False):
        """The return value of _forward_impl once the logits and alphas of the forward are in ``ws``."""
        T = max(decode_lengths)
        philox = isinstance(mask, str)
        # the Philox {seed, call} this forward drew its dropout mask (and sampling coins) from; the backward regenerates the mask
        # from this copy and advances the copy, not the live counter
        dstate = self.dropout_state.clone() if need_grad and (philox or sampling) else None
        if philox or sampling:
            self.dropout_state[1] += 1       # forward-only call: no lo_decoder_backward to advance the Philox call counter
        preds = ws["t"]["logits"][:, :, :self.vocab_size].clone()
        alphas = ws["t"]["alphas"].clone()
        if min(decode_lengths) < T:      # rows that stopped decoding keep zeros (:301-302, :317-318)
            act = torch.arange(T, device=enc.device)[None, :] < torch.tensor(decode_lengths, device=enc.device)[:, None]
            preds = preds * act[:, :, None]
            alphas = alphas * act[:, :, None]
        saved = None
        if need_grad:
            saved = {"entries": [ws], "ws": ws, "enc": enc, "sort_ind": sort_ind, "shape": tuple(encoder_out.shape),
                     "dtype": encoder_out.dtype, "has_do": 0 if mask is None else (2 if philox else 1), "dstate": dstate,
                     "sampling": sampling}
        return (preds, alphas), (caps, decode_lengths, sort_ind), saved

    def _generic_backward_args(self, saved, dpreds):
        """The argument block of a generic-mode lo_decoder_backward of the forward ``saved`` describes: d predictions and the
        forward's Philox state.  Returns (args, the tensors it points at, to be kept referenced until the launches)."""
        ws, enc = saved["ws"], saved["enc"]
        B, R, _ = enc.shape
        T = ws["t"]["hd"].shape[1]
        V = self.vocab_size
        dpred = dpreds.float().contiguous() if dpreds is not None else torch.zeros(B, T, V, device=enc.device)
        # scheduled sampling: ss_prob is the mode flag of the backward (its value is not read), which scatters the embedding
        # gradient by the recorded fed tokens
        a = self.fill_args(ws, enc, B, T, R, saved["has_do"], ss_prob=self._ss_prob if saved.get("sampling") else None)
        dstate = None
        if saved["dstate"] is not None:
            dstate = saved["dstate"].clone()     # lo_decoder_backward advances the counter it is given
            a.dropout_state = dstate.data_ptr()
        a.dpred_ext = dpred.data_ptr()           # also the generic-mode flag
        a.dpred_stride = V
        return a, (dpred, dstate)

    def _scatter_denc(self, saved):
        """d encoder_out in the caller's row order, shape and dtype."""
        denc = saved["ws"]["t"]["denc"]
        dx = torch.empty_like(denc).index_copy_(0, saved["sort_ind"], denc)
        return dx.view(saved["shape"]).to(saved["dtype"])
