"""TensorFlow-flavour decoder — drop-in for the path of model/decoder.py:15-72 (``Decoder(config, n_tok, id_end)``),
model/components/attention_mechanism.py, attention_cell.py, greedy_decoder_cell.py and beam_search_decoder_cell.py on
the sm_90a kernels (csrc/lo_tfdecoder.cuh) through the C ABI (``lo_tfdec_*``).

The reference builds a TF graph; here the same three things the graph offers are methods:
  * ``train_logits(enc, formula)``            -> pred_train  [N,T,V]                      (decoder.py:48-57)
  * ``train_outputs(enc, formula)``           -> (pred_train, alphas [N,T,R]), differentiable: any loss of them trains
                                                 through ``loss.backward()`` (lo_tfdec_backward in its generic mode); with
                                                 ``sampling_prob`` / ``sampling_temperature`` the fed tokens are the model's own
                                                 (scheduled sampling, self-critical training: ``scst``)
  * ``loss_and_backward(enc, formula, len)``  -> masked CE of img2seq.py:68-71 + every gradient (+ d enc)
  * ``decode(enc)``                           -> DecoderOutput(logits=None, ids)          (decoder.py:59-70; greedy ids [N,time],
                                                 beam ids [N,time,beam] like the TF cell before img2seq.py:241 transposes them);
                                                 ``enc`` may be a list of images' encoder outputs of different sizes
``__call__(img, formula, dropout)`` returns ``(train_logits, DecoderOutput)`` like the reference.

Variables keep the TF names and shapes (``embedding_table`` [V,E], ``start_token`` [E], ``att_img.kernel`` [C,A],
``att_h.kernel`` [D,A] (tf.layers.dense inside compute_attention), ``att_beta`` [A], ``lstm.kernel`` [E+O+D,4D], ``lstm.bias``,
``o_W_c``, ``o_W_h``, ``y_W_o``, ``W_{c,h,o}_0``, ``b_{c,h,o}_0``) as views of a flat store whose memory is [out][in]
(K-major for the forward GEMMs).
"""
import collections
import ctypes
import math

import torch
import torch.nn as nn

from . import _lib, decode
from ._lib import TfDecArgs, check, dtype_code, impl_code, stream_ptr
from .kernel_module import kernel_forward, stamp
from .params import FlatStore, LRUCache, ParamHolder, bind_grads

DecoderOutput = collections.namedtuple("DecoderOutput", ("logits", "ids"))      # greedy_decoder_cell.py:5-6
_bind = _lib.lib          # the library with the lo_tfdec_* signatures set (lib() binds them along with the rest)
MAX_ROWS = 512            # decoder rows (images x beam) of one lo_tfdec_* call: the library refuses more


def tf_decoder_specs(V, C, A, D, O, E):
    """Flat order: att_h.kernel^T and o_W_h^T are adjacent (one GEMM projects h_t onto both), the three initial-state
    matrices and their biases likewise, and start_token follows embedding_table (row V of the token table)."""
    return [
        ("att_img.kernel", (A, C)),
        ("att_h.kernel", (A, D)), ("o_W_h", (O, D)),
        ("att_beta", (A,)),
        ("lstm.kernel", (4 * D, E + O + D)), ("lstm.bias", (4 * D,)),
        ("o_W_c", (O, C)), ("y_W_o", (V, O)),
        ("W_c_0", (D, C)), ("W_h_0", (D, C)), ("W_o_0", (O, C)), ("b_c_0", (D,)), ("b_h_0", (D,)), ("b_o_0", (O,)),
        ("embedding_table", (V, E)), ("start_token", (E,)),
    ]


class Decoder(nn.Module):
    def __init__(self, config, n_tok, id_end, device="cuda", precision=None, impl=None, channels=512):
        super().__init__()
        self._config = config
        cell = getattr(config, "attn_cell_config", None) or {}
        self.D = int(cell.get("num_units", 512))
        self.A = int(cell.get("dim_e", 256))
        self.O = int(cell.get("dim_o", 512))
        self.E = int(cell.get("dim_embeddings", 80))
        self.C = channels
        self.V = int(n_tok)
        self._n_tok, self._id_end = int(n_tok), int(id_end)
        self.decoding = getattr(config, "decoding", "greedy")
        if self.decoding not in ("greedy", "beam_search"):
            raise NotImplementedError("decoding=%r" % (self.decoding,))
        self._tiles = 1 if self.decoding == "greedy" else int(getattr(config, "beam_size", 2))        # decoder.py:22
        # diversity penalty of beam_search_decoder_cell.py:258-287 (off in the shipped config: model.json:15-16 -> gamma 1, prob 0)
        self.div_gamma = float(getattr(config, "div_gamma", 1) or 1)
        self.div_prob = float(getattr(config, "div_prob", 0) or 0)
        # length and coverage penalties of GNMT (lo_beam_penalty); 0, the reference's search, when the config has none
        self.length_penalty, self.coverage_penalty = decode.penalty_weights(getattr(config, "length_penalty", 0) or 0,
                                                                            getattr(config, "coverage_penalty", 0) or 0)
        self._div_state = None
        self.max_length_formula = int(getattr(config, "max_length_formula", 150))
        self.precision = precision or getattr(config, "precision", "bf16")
        self.impl = impl if impl is not None else getattr(config, "conv_impl", "tc" if self.precision == "bf16" else "simt")
        self.tdtype = torch.float32 if self.precision == "fp32" else torch.bfloat16
        self.store = FlatStore(tf_decoder_specs(self.V, self.C, self.A, self.D, self.O, self.E), device,
                               bf16_shadow=(self.precision == "bf16"))
        S = self.store
        bind = ParamHolder.bind
        for holder, sname in (("att_img", "att_img.kernel"), ("att_h", "att_h.kernel")):
            h = ParamHolder()
            h.bind("kernel", S, sname, permute=(1, 0))
            setattr(self, holder, h)
        self.lstm = ParamHolder()
        self.lstm.bind("kernel", S, "lstm.kernel", permute=(1, 0))
        self.lstm.bind("bias", S, "lstm.bias")
        for n in ("o_W_c", "o_W_h", "y_W_o", "W_c_0", "W_h_0", "W_o_0"):
            bind(self, n, S, n, permute=(1, 0))
        for n in ("att_beta", "b_c_0", "b_h_0", "b_o_0", "embedding_table", "start_token"):
            bind(self, n, S, n)
        self.reset_parameters()
        self._ws = LRUCache()     # bounded: see params.LRUCache
        # sampling (train_outputs(..., sampling_prob=p)): the device scalars p and tau the kernels read (created on first use), the
        # Philox {seed, call} of the coins and Gumbel uniforms (one call per sampling forward), the tokens fed by the last forward
        # [N, T], and injected coins [N, T] / Gumbel uniforms [N, T, V] for parity tests (None: Philox)
        self._ss_prob = self._ss_temp = None
        self.ss_state = torch.tensor([int(torch.initial_seed()) & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64, device=device)
        self.last_fed_tokens = None
        self._ss_u = self._ss_gu = None

    def seed_sampling(self, seed, call=0):
        """Seeds the Philox stream of the sampling coins and Gumbel uniforms; every sampling forward uses up one ``call``."""
        self.ss_state.copy_(torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, int(call)], dtype=torch.int64))

    @staticmethod
    def check_sampling(sampling_prob, sampling_temperature):
        """The argument checks of DecoderWithAttention.forward."""
        if not 0.0 <= sampling_prob <= 1.0:
            raise ValueError("sampling_prob must lie in [0, 1] (got %r)" % (sampling_prob,))
        if not (sampling_temperature >= 0.0 and math.isfinite(sampling_temperature)):
            raise ValueError("sampling_temperature must be a finite tau >= 0 (got %r)" % (sampling_temperature,))
        if sampling_temperature > 0.0 and sampling_prob == 0.0:
            raise ValueError("sampling_temperature needs sampling_prob > 0: it sets how the fed tokens are drawn")

    def sampling_scalars(self, sampling_prob, sampling_temperature=0.0):
        """(p, tau) as the device scalars run_forward takes, None for off (p = 0: teacher forcing; tau = 0: the argmax)."""
        self.check_sampling(sampling_prob, sampling_temperature)
        ss = tau = None
        if sampling_prob > 0.0:
            if self._ss_prob is None:
                self._ss_prob = torch.zeros((), dtype=torch.float32, device=self.store.device)
            ss = self._ss_prob
            ss.fill_(sampling_prob)
        if sampling_temperature > 0.0:
            if self._ss_temp is None:
                self._ss_temp = torch.zeros((), dtype=torch.float32, device=self.store.device)
            tau = self._ss_temp
            tau.fill_(sampling_temperature)
        return ss, tau

    # tf.get_variable / tf.layers.dense default: glorot_uniform; LSTMCell bias zeros; embeddings decoder.py:98-105
    def reset_parameters(self):
        def glorot_(p, fan_in, fan_out):
            lim = math.sqrt(6.0 / (fan_in + fan_out))
            p.uniform_(-lim, lim)

        with torch.no_grad():
            for p in (self.att_img.kernel, self.att_h.kernel, self.lstm.kernel, self.o_W_c, self.o_W_h, self.y_W_o, self.W_c_0,
                      self.W_h_0, self.W_o_0):
                glorot_(p, p.shape[0], p.shape[1])
            glorot_(self.att_beta, self.A, 1)
            for p in (self.b_c_0, self.b_h_0, self.b_o_0):
                glorot_(p, p.shape[0], p.shape[0])
            self.lstm.bias.zero_()
            for p in (self.embedding_table, self.start_token):
                p.uniform_(-1.0, 1.0)
                p.copy_(torch.nn.functional.normalize(p, dim=-1))

    def load_tf_variables(self, d):
        """d: name -> tensor in the TF shapes (module docstring); ``att_beta`` may be [A,1]."""
        sd = self.state_dict()
        with torch.no_grad():
            for k, v in d.items():
                sd[k].copy_(v.reshape(sd[k].shape))

    # ---------------------------------------------------------------------------------------------
    def _args(self, enc, B, T, R, rows_per_img=1, decode=False, ws=None):
        """Args and workspace of one shape.  Decoding has workspaces of its own, so a decode never overwrites the saved state of
        a teacher-forced pass whose autograd backward is still to run (Decoder.forward runs both).  ``ws``: a workspace of the
        caller's (ragged_workspace) instead of the shape's own."""
        L = _lib.lib()
        key = (B, T, R, rows_per_img, "decode") if decode else (B, T, R, rows_per_img)
        ws = self._ws.get(key) if ws is None else ws
        dev = self.store.device
        if ws is None:
            ws = {"ldl": (self.V + 63) // 64 * 64}
            ws["logits"] = torch.zeros(T, B, ws["ldl"], dtype=torch.float32, device=dev)
            ws["alphas"] = torch.zeros(B, T, R, dtype=torch.float32, device=dev)
            ws["loss"] = torch.zeros(4, dtype=torch.float32, device=dev)
            ws["denc"] = torch.zeros(B // rows_per_img, R, self.C, dtype=torch.float32, device=dev)
            ws["formula"] = torch.zeros(B, T, dtype=torch.int64, device=dev)
            ws["lengths"] = torch.zeros(B, dtype=torch.int32, device=dev)
            self._ws[key] = ws
        stamp(ws)              # every caller overwrites the forward state: a pending autograd backward of it must refuse to run
        S = self.store
        a = TfDecArgs()
        a.B, a.T, a.R, a.C, a.A, a.D, a.O, a.E, a.V = B, T, R, self.C, self.A, self.D, self.O, self.E, self.V
        a.dt = dtype_code(self.precision)
        a.impl = impl_code(self.impl, self.precision)
        a.ldl = ws["ldl"]
        a.rows_per_img = rows_per_img
        a.enc = enc.data_ptr()
        a.formula, a.formula_stride = ws["formula"].data_ptr(), ws["formula"].stride(0)
        a.lengths = ws["lengths"].data_ptr()
        W, F, G = (lambda n: S.w(n).data_ptr()), (lambda n: S.f32(n).data_ptr()), (lambda n: S.g(n).data_ptr())
        a.w_img, a.w_cat2, a.beta = W("att_img.kernel"), W("att_h.kernel"), F("att_beta")
        a.w_lstm, a.b_lstm, a.w_oc, a.w_y = W("lstm.kernel"), F("lstm.bias"), W("o_W_c"), W("y_W_o")
        a.w_init, a.b_init, a.emb = W("W_c_0"), F("b_c_0"), W("embedding_table")
        a.g_w_img, a.g_w_cat2, a.g_beta = G("att_img.kernel"), G("att_h.kernel"), G("att_beta")
        a.g_w_lstm, a.g_b_lstm, a.g_w_oc, a.g_w_y = G("lstm.kernel"), G("lstm.bias"), G("o_W_c"), G("y_W_o")
        a.g_w_init, a.g_b_init, a.g_emb = G("W_c_0"), G("b_c_0"), G("embedding_table")
        for k in ("logits", "alphas", "loss", "denc"):
            setattr(a, k, ws[k].data_ptr() if ws[k] is not None else None)
        if "ws" not in ws:
            ws["ws"] = torch.zeros(int(L.lo_tfdec_workspace_bytes(ctypes.byref(a))), dtype=torch.uint8, device=dev)
        a.ws = ws["ws"].data_ptr()
        ws["args"] = a
        return L, ws, a

    def _enc(self, enc):
        if not enc.is_cuda:
            raise _lib.LatexOcrB200Error("Decoder runs on CUDA tensors only (no CPU fallback)")
        if enc.dim() == 4:                                   # attention_mechanism.py:21-26: [N,H,W,C] -> [N,H*W,C]
            enc = enc.reshape(enc.shape[0], enc.shape[1] * enc.shape[2], enc.shape[3])
        return enc.to(self.tdtype).contiguous()

    def _keep(self, a, ws, keep_h, keep_o, T, B):
        """Optional dropout multipliers [N,T,D] / [N,T,O] (tf.nn.dropout semantics: 0 or 1/keep_prob) -> time-major."""
        for name, k, width in (("keep_h", keep_h, self.D), ("keep_o", keep_o, self.O)):
            if k is None:
                continue
            ws[name] = k.to(self.store.device, torch.float32).permute(1, 0, 2).contiguous()
            assert ws[name].shape == (T, B, width)
            setattr(a, name, ws[name].data_ptr())

    def run_forward(self, enc, formula, lengths=None, keep_h=None, keep_o=None, n_words=None, ss_prob=None, ss_temp=None):
        """enc [N,R,C] or [N,H,W,C]; formula int64 [N,T]; lengths [N] (incl. END) enables the loss.  Returns the workspace dict
        (``logits`` [T,N,ldl] time-major, ``alphas`` [N,T,R], ``loss``).  ss_prob / ss_temp: None, or the device scalars of
        sampling_scalars: the tokens fed land in ``ws["fed"]`` [N,T] (lo_tfdec_args.ss_prob), and the call uses up one Philox call
        of ``ss_state``."""
        enc = self._enc(enc)
        B, R, _ = enc.shape
        T = formula.shape[1]
        self.store.refresh_shadow()
        L, ws, a = self._args(enc, B, T, R)
        ws["enc"] = enc
        ws["formula"].copy_(formula)
        with_loss = lengths is not None
        if with_loss:
            lens = torch.as_tensor(lengths, dtype=torch.int32)
            ws["lengths"].copy_(lens)
            # data parallel: n_words = token count of the GLOBAL batch, so that summing rank gradients gives the global mean
            a.inv_n_words = 1.0 / float(n_words if n_words is not None else int(lens.sum()))
        self._keep(a, ws, keep_h, keep_o, T, B)
        if ss_prob is not None:
            if ws.get("fed") is None:
                ws["fed"] = torch.zeros(B, T, dtype=torch.int64, device=self.store.device)
            a.ss_prob, a.fed, a.ss_state = ss_prob.data_ptr(), ws["fed"].data_ptr(), self.ss_state.data_ptr()
            for name, inj, shape, on in (("ss_u", self._ss_u, (B, T), True), ("ss_gu", self._ss_gu, (B, T, self.V), ss_temp is not None)):
                if inj is not None and on:
                    ws[name] = inj.to(self.store.device, torch.float32).contiguous()
                    assert ws[name].shape == shape
                    setattr(a, name, ws[name].data_ptr())
            if ss_temp is not None:
                a.ss_temp = ss_temp.data_ptr()
        check(L.lo_tfdec_forward(ctypes.byref(a), 1 if with_loss else 0, stream_ptr()))
        if ss_prob is not None:
            self.ss_state[1] += 1            # the next sampling forward draws from a new Philox call
        return ws

    def run_backward(self, ws):
        check(_lib.lib().lo_tfdec_backward(ctypes.byref(ws["args"]), stream_ptr()))
        return ws["denc"]

    def train_logits(self, enc, formula, keep_h=None, keep_o=None):
        with torch.no_grad():
            ws = self.run_forward(enc, formula, None, keep_h, keep_o)
            return ws["logits"][:, :, :self.V].permute(1, 0, 2).contiguous()

    def train_outputs(self, enc, formula, keep_h=None, keep_o=None, sampling_prob=0.0, sampling_temperature=0.0):
        """Teacher-forced pass: (logits [N,T,V], alphas [N,T,R]).  With grad mode on and ``enc`` or a parameter requiring grad, an
        autograd graph is recorded: both outputs are differentiable (any loss of them), d enc comes back in ``enc``'s shape and
        dtype, and the backward runs lo_tfdec_backward in its generic mode with the same keep masks.  The outputs are the same
        either way.

        ``sampling_prob`` = p > 0: scheduled sampling (Bengio et al. 2015) inside the CUDA time loop.  Every step predicts: step t
        predicts ``formula[:, t]`` and step t+1 consumes ``fed[b][t]``, which is the lowest-index argmax of the returned logits
        ``[b, t]`` where a coin u ~ U[0,1) is below p, ``formula[b][t]`` otherwise (step 0 consumes the start token).  The coins come
        from Philox keyed by ``ss_state`` (``philox.sampling_uniforms``; one call per sampling forward, also without grad;
        ``seed_sampling`` reproduces them).  ``last_fed_tokens`` holds fed [N,T]; its last column is consumed by no step.  The
        choice is not differentiated: the backward is teacher forcing on fed, and a loss's targets stay ``formula``.
        ``sampling_temperature`` = tau > 0 (with p > 0): a step that samples feeds a draw from softmax(logits / tau) (Gumbel-max,
        ``philox.gumbel_uniforms``) instead of the argmax; with p = 1 the call samples whole formulas and a policy-gradient loss
        of the outputs trains through ``loss.backward()`` (``scst``).  p = 0 (the default) is the teacher-forced path unchanged."""
        return kernel_forward(self, (enc, formula, keep_h, keep_o, float(sampling_prob), float(sampling_temperature or 0.0)), (enc,))[0]

    def _forward_impl(self, enc, formula, keep_h, keep_o, sampling_prob=0.0, sampling_temperature=0.0, need_grad=False):
        """((logits, alphas), None, what the backward of this call needs or None)."""
        ss, tau = self.sampling_scalars(sampling_prob, sampling_temperature)
        ws = self.run_forward(enc, formula, None, keep_h, keep_o, ss_prob=ss, ss_temp=tau)
        self.last_fed_tokens = (ws["fed"] if ss is not None else ws["formula"]).clone()
        logits = ws["logits"][:, :, :self.V].permute(1, 0, 2).contiguous()
        alphas = ws["alphas"].clone()
        saved = None
        if need_grad:
            # ws["args"] points at ws["enc"] and the keep masks of this call; holding them keeps them alive even if the workspace
            # leaves the cache
            saved = {"entries": [ws], "ws": ws, "args": ws["args"], "enc": ws["enc"],
                     "keep": (ws["keep_h"] if keep_h is not None else None, ws["keep_o"] if keep_o is not None else None),
                     "shape": tuple(enc.shape), "dtype": enc.dtype}
        return (logits, alphas), None, saved

    def _backward_impl(self, saved, dlogits, dalphas, need):
        """lo_tfdec_backward in its generic mode: returns (d enc in the caller's shape and dtype,)."""
        ws = saved["ws"]
        B, T, R = ws["alphas"].shape
        dev = self.store.device
        dl = dlogits.float().contiguous() if dlogits is not None else torch.zeros(B, T, self.V, device=dev)
        dal = dalphas.float().contiguous() if dalphas is not None else None
        a = TfDecArgs.from_buffer_copy(saved["args"])
        a.dlogits_ext, a.dlogits_stride = dl.data_ptr(), self.V
        a.dalpha_ext = dal.data_ptr() if dal is not None else None
        check(_lib.lib().lo_tfdec_backward(ctypes.byref(a), stream_ptr()))
        return (ws["denc"].reshape(saved["shape"]).to(saved["dtype"], copy=True),)

    def loss_and_backward(self, enc, formula, lengths, keep_h=None, keep_o=None, n_words=None, sampling_prob=0.0):
        """Returns (loss tensor [4] on the device: mean CE, mean CE, 0, n_words; d loss / d enc [N,R,C] fp32).  Parameter
        gradients land in ``self.store.grad`` (the ``.grad`` of every parameter).  ``sampling_prob`` = p > 0: scheduled sampling
        as in train_outputs (the CE targets stay ``formula``); ``last_fed_tokens`` is then the step's fed buffer [N,T]."""
        bind_grads(self, self.store)             # autograd use or zero_grad(set_to_none=True) may have re-pointed p.grad
        with torch.no_grad():
            ss, _ = self.sampling_scalars(float(sampling_prob))
            ws = self.run_forward(enc, formula, lengths, keep_h, keep_o, n_words, ss_prob=ss)
            self.last_fed_tokens = ws["fed"] if ss is not None else None
            denc = self.run_backward(ws)
            return ws["loss"], denc

    def ragged_workspace(self, B, T, R, n_regions):
        """Decode workspace for images of different sizes (lo_tfdec_args.reg_off): the packed encoder output ``enc`` [regions, C],
        the region offsets ``reg_off`` / ``reg_off_host`` and every per-row buffer, sized by capacity (rows B, steps T, largest
        region count R, total regions; decode.ragged_cache)."""
        def build(B, T, R, n_regions):
            dev = self.store.device
            ldl = (self.V + 63) // 64 * 64
            z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device=dev)
            ws = {"ldl": ldl,
                  "logits": z(B, ldl),                    # decoding writes one step's logits, [B][V]
                  "alphas": z(B * T * R),                 # [B][T][R] of each call's own B, T and R
                  "loss": z(4), "denc": None, "formula": z(B, T, dtype=torch.int64), "lengths": z(B, dtype=torch.int32),
                  "enc": z(n_regions, self.C, dtype=self.tdtype),
                  "reg_off": z(B + 1, dtype=torch.int32), "reg_off_host": (ctypes.c_int32 * (B + 1))()}
            # sizes the kernel workspace: every region of it grows with B, T, R and B / rows_per_img, so any call that fits the
            # capacity fits in it (the beam size is the decoder's own, fixed at construction)
            self._args(ws["enc"], B, T, R, rows_per_img=self._tiles, ws=ws)
            return ws
        return decode.ragged_cache(self._ws, (B, T, R, n_regions), build)

    def packed_workspace(self, counts, steps, rows_per_img=None):
        """The ragged workspace of one decode call over images of ``counts`` regions (in the order they are decoded).  The caller
        writes image i's encoder output into ``ws["enc"][off[i]:off[i+1]]`` (``ws["off"]``) and then calls decode_packed.
        ``rows_per_img``: the rows of each image (default: the beam size; sample() passes its sample count)."""
        N = len(counts)
        rpi = self._tiles if rows_per_img is None else int(rows_per_img)
        if N == 0:
            raise ValueError("no images")
        if min(counts) < 1:
            raise ValueError("an image has no encoder region")
        if N * rpi > MAX_ROWS:
            raise ValueError("%d images x %d rows exceed the %d rows of one decode call" % (N, rpi, MAX_ROWS))
        off = decode.region_offsets(counts)
        # the kernel workspace is sized for B / beam images, so a call of fewer rows per image asks for that many more rows
        ws = self.ragged_workspace(N * max(rpi, self._tiles), steps, max(counts), off[-1])
        ws["counts"], ws["off"] = [int(n) for n in counts], off
        return ws

    def decode_packed(self, ws, steps, div_u=None, return_attention=False, return_log_probs=False, finalize="reference",
                      return_scores=False, brackets=None):
        """decode() over the images packed in ``ws`` by packed_workspace: every image attends over its own regions only."""
        if finalize not in ("reference", "backtrack"):
            raise NotImplementedError("finalize must be 'reference' or 'backtrack'")
        if self.decoding != "greedy":
            decode.refuse_reference_finalize(brackets, finalize)
        counts = ws["counts"]
        N, beam = len(counts), self._tiles
        R = max(counts)
        self.store.refresh_shadow()
        with torch.no_grad():
            L, ws, a = self._args(ws["enc"], N * beam, steps, R, rows_per_img=beam, ws=ws)
            decode.set_region_offsets(a, ws["reg_off_host"], ws["reg_off"], ws["off"])
            alphas = ws["alphas"][:N * beam * steps * R].view(N * beam, steps, R) if return_attention else None
            out = self._run_decode(L, a, N, steps, div_u, alphas, return_log_probs, finalize, return_scores, brackets)
            if alphas is None:
                return out
            att = out[-1]
            if self.decoding == "greedy":
                return out[:-1] + ([att[i, :, :counts[i]].clone() for i in range(N)],)
            return out[:-1] + ([att[i, :, :, :counts[i]].clone() for i in range(N)],)

    def decode(self, enc, max_steps=None, div_u=None, return_attention=False, return_log_probs=False, finalize="reference",
               return_scores=False, brackets=None):
        """dynamic_decode(decoder_cell, max_length_formula + 1) (decoder.py:70): at most max_length_formula + 2 steps, stops when
        every row / beam has emitted END.  Returns DecoderOutput(logits=None, ids).  ``div_u`` (tests): injected uniforms
        [steps, N*beam, V] for the diversity penalty; ``return_log_probs`` (beam search): also the log-probs of the hypotheses
        [N, beam]; ``return_attention``: also the attention weights (the tensor attention_mechanism.py:96-121 hands to
        visualize_attention.py), after the log-probs: greedy [N, steps, R], beam search [N, beam, steps, R].
        ``finalize`` (beam search): 'reference' returns the reference's identity finalize (ids[:, t, s] is what slot s chose at step
        t) and the rows slot s computed, what visualize_attention.py draws for s = 0; 'backtrack' returns lineage-consistent
        hypotheses, ids [N, steps, beam] followed back from each final slot, and the attention under which each of their tokens
        was chosen (the rows of a teacher-forced pass over the hypothesis).
        The search ranks hypotheses with the length and coverage penalties of the config's ``length_penalty`` /
        ``coverage_penalty`` (lo_beam_penalty; 0: the reference's search); the log-probs stay the raw sums, and
        ``return_scores`` (beam search) also returns the ranking scores [N, beam], after the log-probs.

        ``enc`` [N,R,C] / [N,H,W,C], or a list of the encoder outputs of images of different sizes, each [H_i,W_i,C] or [R_i,C]:
        the list is decoded in one time loop in which every image attends over its own regions only (lo_tfdec_args.reg_off), so
        an image's ids do not depend on the other images of the call.  Ids come back in input order, image i draws the rows
        [i*beam, (i+1)*beam) of ``div_u``, and ``return_attention`` gives a list of [steps, R_i] (greedy) or [beam, steps, R_i]
        tensors.

        ``brackets``: a decode.BracketRule (lo_tfdec_greedy_brackets / lo_tfdec_beam_brackets): every formula, and every beam
        hypothesis under ``finalize='backtrack'``, nests its brackets and closes them; beam search refuses it with 'reference'."""
        if finalize not in ("reference", "backtrack"):
            raise NotImplementedError("finalize must be 'reference' or 'backtrack'")
        if self.decoding != "greedy":
            decode.refuse_reference_finalize(brackets, finalize)
        steps = int(max_steps) if max_steps is not None else self.max_length_formula + 2
        if isinstance(enc, (list, tuple)):
            encs = [self._enc_regions(e) for e in enc]
            ws = self.packed_workspace([e.shape[0] for e in encs], steps)
            off = ws["off"]
            for i, e in enumerate(encs):
                ws["enc"][off[i]:off[i + 1]].copy_(e)
            return self.decode_packed(ws, steps, div_u, return_attention, return_log_probs, finalize, return_scores, brackets)
        enc = self._enc(enc)
        N, R, _ = enc.shape
        self.store.refresh_shadow()
        with torch.no_grad():
            L, ws, a = self._args(enc, N * self._tiles, steps, R, rows_per_img=self._tiles, decode=True)
            ws["enc"] = enc
            return self._run_decode(L, a, N, steps, div_u, ws["alphas"] if return_attention else None, return_log_probs, finalize,
                                    return_scores, brackets)

    def sample(self, enc, n_samples=8, temperature=1.0, top_k=0, top_p=1.0, max_steps=None, u=None, seed=None,
               return_attention=False, brackets=None):
        """Sampling decode (lo_tfdec_sample): ``n_samples`` formulas per image, each step's token drawn from softmax(logits /
        ``temperature``) restricted by ``top_k`` / ``top_p``, as decode.sample_decode documents.  ``enc`` as in decode(): a batch
        [N,R,C] / [N,H,W,C] or a list of the encoder outputs of images of different sizes.  Returns (ids [N, n_samples, steps],
        log_probs [N, n_samples]) on the device, ids in input order, and with ``return_attention`` the attention weights [N,
        n_samples, steps, R] (a list of [n_samples, steps, R_i] for a list).  ``seed``: a new Philox stream at that seed, else the
        decoder's own, which every call advances; ``u`` (tests): injected uniforms [steps, N * n_samples, V], image i drawing the
        rows [i * n_samples, (i + 1) * n_samples).  ``brackets``: a decode.BracketRule (lo_tfdec_sample_brackets), as
        decode.sample_decode documents."""
        n, tau, k, p = decode.sampling_settings(n_samples, temperature, top_k, top_p, self.V)
        steps = int(max_steps) if max_steps is not None else self.max_length_formula + 2
        dev = self.store.device
        self.store.refresh_shadow()
        counts = None
        if isinstance(enc, (list, tuple)):
            encs = [self._enc_regions(e) for e in enc]
            counts = [e.shape[0] for e in encs]
            ws = self.packed_workspace(counts, steps, n)
            off = ws["off"]
            for i, e in enumerate(encs):
                ws["enc"][off[i]:off[i + 1]].copy_(e)
            N, R = len(encs), max(counts)
        else:
            enc = self._enc(enc)
            N, R, _ = enc.shape
            ws = None
        with torch.no_grad():
            state = decode.sample_state(self, seed, dev) if u is None else None
            if counts is None:
                L, ws, a = self._args(enc, N * n, steps, R, rows_per_img=n, decode=True)
                ws["enc"] = enc
            else:
                L, ws, a = self._args(ws["enc"], N * n, steps, R, rows_per_img=n, ws=ws)
                decode.set_region_offsets(a, ws["reg_off_host"], ws["reg_off"], ws["off"])

            br, keep = decode.bracket_args(brackets, self._id_end, self.V, a.B, steps, dev)

            def call(s, tokens, fin):
                if br is not None:
                    return L.lo_tfdec_sample_brackets(ctypes.byref(a), ctypes.byref(s), self._id_end, steps, tokens, fin,
                                                      ctypes.byref(br), stream_ptr())
                return L.lo_tfdec_sample(ctypes.byref(a), ctypes.byref(s), self._id_end, steps, tokens, fin, stream_ptr())
            ids, logp = decode.run_sample(call, N, n, steps, tau, k, p, self.V, state, dev, u)
            if not return_attention:
                return ids, logp
            att = ws["alphas"].view(-1)[:N * n * steps * R].view(N, n, steps, R)[:, :, :ids.shape[2]].clone()
            if counts is not None:
                att = [att[i, :, :, :counts[i]].clone() for i in range(N)]
            return ids, logp, att

    def _enc_regions(self, e):
        """one image's encoder output of a list -> [R_i, C] on the device"""
        if not e.is_cuda:
            raise _lib.LatexOcrB200Error("Decoder runs on CUDA tensors only (no CPU fallback)")
        if e.dim() == 3:
            e = e.reshape(e.shape[0] * e.shape[1], e.shape[2])
        if e.dim() != 2 or e.shape[1] != self.C:
            raise ValueError("each image's encoder output must be [H,W,%d] or [R,%d] (got shape %s)" % (self.C, self.C, tuple(e.shape)))
        return e

    def _run_decode(self, L, a, N, steps, div_u, alphas, return_log_probs, finalize="reference", return_scores=False,
                    brackets=None):
        """The greedy or beam decode of the filled args ``a`` (N images); ``alphas``: the attention rows [B, steps, R] of the call
        (attention export) or None; ``brackets``: a decode.BracketRule or None."""
        dev = self.store.device
        br, keep = decode.bracket_args(brackets, self._id_end, self.V, a.B, steps, dev, self._tiles)
        if self.decoding == "greedy":
            def greedy(tokens, fin):
                if br is not None:
                    return L.lo_tfdec_greedy_brackets(ctypes.byref(a), self._id_end, steps, tokens, fin, ctypes.byref(br), stream_ptr())
                return L.lo_tfdec_greedy(ctypes.byref(a), self._id_end, steps, tokens, fin, stream_ptr())
            ids = decode.run_greedy(greedy, N, steps, dev)
            if alphas is not None:
                return DecoderOutput(None, ids), alphas[:, :ids.shape[1]].float().clone()
            return DecoderOutput(None, ids)
        div_on = not (self.div_gamma == 1 or self.div_prob == 0)
        state = None
        if div_on and div_u is None:
            if self._div_state is None:
                self._div_state = torch.tensor([torch.initial_seed() & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64, device=dev)
            self._div_state[1] += 1                                  # a new Philox stream per decode call
            state = self._div_state.data_ptr()

        alpha, beta = self.length_penalty, self.coverage_penalty
        pen = None
        if alpha != 0 or beta > 0 or return_scores:
            pen, pen_t = decode.beam_penalty(alpha, beta, a.B, a.R, steps, self._tiles, dev)

        def call(ids, parents, fin, logp, u):
            args = (ctypes.byref(a), self._id_end, steps, ids, parents, fin, logp, self.div_gamma, self.div_prob, u, state)
            if br is not None:
                return L.lo_tfdec_beam_brackets(*args, ctypes.byref(pen) if pen is not None else None, ctypes.byref(br), stream_ptr())
            if pen is not None:
                return L.lo_tfdec_beam_pen(*args, ctypes.byref(pen), stream_ptr())
            return L.lo_tfdec_beam_div(*args, stream_ptr())
        ids, parents, logp = decode.run_beam(call, N, self._tiles, steps, self.V, dev, div_u if div_on else None)
        # finalize (beam_search_decoder_cell.py:189-250) gathers with the unchanged initial parents -> identity (SURVEY §8-A.3)
        att = None
        if alphas is not None or finalize == "backtrack":
            hyp, att = decode.beam_hypotheses(ids, parents, finalize, a, alphas)
            if finalize == "backtrack":
                ids = hyp.permute(0, 2, 1).contiguous()
        out = ((DecoderOutput(None, ids),) + ((logp,) if return_log_probs else ()) + ((pen_t["scores"],) if return_scores else ())
               + ((att,) if alphas is not None else ()))
        return out if len(out) > 1 else out[0]

    def forward(self, img, formula=None, dropout=1.0):
        """Decoder.__call__(img, formula, dropout) (decoder.py:24): (pred_train, pred_test).  dropout is the TF keep_prob; the
        shipped training config uses 1 (training.json:7) — other values draw masks here.  pred_train comes from train_outputs, so
        it is differentiable under the same rule (its backward reuses the masks drawn here)."""
        keep_h = keep_o = None
        train = None
        if formula is not None:
            if dropout is not None and float(dropout) < 1.0:
                N, T = formula.shape
                kp = float(dropout)
                dev = self.store.device
                keep_h = (torch.rand(N, T, self.D, device=dev) < kp).float() / kp
                keep_o = (torch.rand(N, T, self.O, device=dev) < kp).float() / kp
            train = self.train_outputs(img, formula, keep_h, keep_o)[0]
        return train, self.decode(img)
