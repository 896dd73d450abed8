"""Img2SeqModel — the trainer surface of model/img2seq_torch.py:64-172 + model/base_torch.py:45-206
(build_train / getLoss / _run_train_epoch / train) on the H100-native encoder and decoder.

``getLoss`` keeps the reference semantics exactly (img2seq_torch.py:136-172): every row's caption
length is the padded length (:144), targets are captions[:, 1:] (:147), loss = CE(mean over packed
positions, PADs included) + 1.0 * mean((1 - sum_t alpha)^2) (:151-159), backward, Adam step on the
decoder then the encoder (:162-170), returns ``-loss`` (:172).  The ``lr`` and ``dropout`` arguments
are ignored exactly like the reference ignores them (SURVEY.md quirk Q3).
"""
import ctypes
import math
import os
import time

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr, stream_ptr
from .decoder import DecoderWithAttention
from .encoder import EncoderCNN
from .params import LRUCache, bind_grads


def bracket_rule(config, vocab):
    """The decode.BracketRule of ``config.balanced_brackets`` (default off: None), built once per vocabulary from its id_to_tok
    table with BracketRule.latex and kept on the vocabulary."""
    if not getattr(config, "balanced_brackets", False):
        return None
    from . import decode
    if vocab is None or getattr(vocab, "id_to_tok", None) is None:
        raise ValueError("balanced_brackets needs a vocabulary with an id_to_tok table")
    rule = getattr(vocab, "_bracket_rule", None)
    if rule is None:
        rule = decode.BracketRule.latex(vocab.id_to_tok)
        vocab._bracket_rule = rule
    return rule


class Img2SeqModel:
    def __init__(self, config, dir_output=None, vocab=None, device=None, precision=None, impl=None, n_tok=None):
        self._config = config
        self._dir_output = dir_output
        self._vocab = vocab
        dev = device or getattr(config, "device", "cuda")
        if not str(dev).startswith("cuda"):
            raise _lib.LatexOcrB200Error("latex_ocr_b200 runs on CUDA devices only (device=%r)" % (dev,))
        self.device = torch.device(dev)
        self.precision = precision or getattr(config, "precision", "bf16")
        # kernels: "tc" = wgmma/TMA convolutions and GEMMs (bf16 storage only), "simt" = CUDA-core twins (fp32 tight-parity mode)
        self.impl = impl or getattr(config, "impl", "tc" if self.precision == "bf16" else "simt")
        self._n_tok = n_tok if n_tok is not None else (vocab.n_tok if vocab is not None else None)
        self.encoder = None
        self.decoder = None
        self.use_graph = bool(getattr(config, "cuda_graph", False))
        self._graphs = LRUCache()  # captured train-step graphs, one per (shapes, mode): bounded like the workspaces
        self.dist = None          # set by latex_ocr_b200.dist.attach(model)
        self.lr = float(getattr(config, "lr_init", 1e-3))
        # scheduled sampling in the fused step: p (host copy) and the device scalar the kernels read (created when p first > 0)
        self.sampling_prob = 0.0
        self._ss_prob_dev = None
        self.set_sampling_prob(getattr(config, "sampling_prob", 0.0) or 0.0)
        # self-critical training in the fused step: tau (host copy; 0 = cross-entropy) and the device scalars the kernels read
        self.scst_temperature = 0.0
        self._scst_temp_dev = None
        self._scst_one = None

    # --- model/base_torch.py:45-71 -------------------------------------------------------------
    def build_train(self, config=None):
        config = config or self._config
        self.getModel("Img2Seq")
        self.getOptimizer(getattr(config, "lr_method", "adam"), float(getattr(config, "lr_init", 1e-3)))
        return self

    def build_pred(self, config=None):
        self.getModel("Img2Seq")
        return self

    def getModel(self, model_name="Img2Seq"):
        """img2seq_torch.py:69-83 (only the Img2Seq branch is on the hot path)."""
        if model_name != "Img2Seq":
            raise NotImplementedError("model_name=%r: only 'Img2Seq' is implemented" % model_name)
        self.encoder = EncoderCNN(self._config, device=self.device, precision=self.precision, impl=self.impl)
        self.decoder = DecoderWithAttention(attention_dim=512, embed_dim=512, decoder_dim=512, vocab_size=self._n_tok,
                                            dropout=0.5, device=self.device, precision=self.precision, impl=self.impl)
        return self

    def getOptimizer(self, lr_method="adam", lr=0.001):
        """img2seq_torch.py:85-88: two Adam optimisers with torch defaults (one fused launch each)."""
        if str(lr_method).lower() != "adam":
            raise NotImplementedError("lr_method=%r: the torch path of the reference always builds Adam" % lr_method)
        self.lr = float(lr)
        self.encoder.store.ensure_adam(lr)
        self.decoder.store.ensure_adam(lr)

    def set_lr(self, lr):
        """Learning rate of both fused Adam optimisers (a device scalar read by the kernel: works under graph replay)."""
        self.lr = float(lr)
        self.encoder.store.set_lr(lr)
        self.decoder.store.set_lr(lr)

    def set_sampling_prob(self, p):
        """Scheduled sampling (Bengio et al. 2015) in the fused train step: from the next step on, each decoder step t >= 1 feeds
        the model's own argmax prediction of step t-1 with probability p instead of the teacher token (DecoderWithAttention.forward
        documents the rule).  p is a device scalar read by the kernels, so a captured step graph picks up a new p without
        re-capture; p = 0 runs the teacher-forced step (its own graph).  No schedule is built in: set p per epoch.  The tokens fed
        by the last step are ``self.decoder.last_fed_tokens`` (a view of the step's buffer)."""
        p = float(p)
        if not 0.0 <= p <= 1.0:
            raise ValueError("sampling_prob must lie in [0, 1] (got %r)" % (p,))
        if p > 0.0 and getattr(self, "scst_temperature", 0.0) > 0.0:
            raise _lib.LatexOcrB200Error("scheduled sampling and self-critical training exclude each other: call "
                                         "set_self_critical(None) first")
        self.sampling_prob = p
        if p > 0.0:
            if self._ss_prob_dev is None:
                self._ss_prob_dev = torch.zeros((), dtype=torch.float32, device=self.device)
            self._ss_prob_dev.fill_(p)

    def set_self_critical(self, temperature):
        """Self-critical sequence training (SCST; Rennie et al. 2017) in the fused train step.  ``temperature`` = tau > 0: from the
        next step on, ``train_step`` / ``getLoss`` / ``_run_train_epoch`` / ``train`` sample one formula per image from
        softmax(logits / tau) inside the CUDA time loop, score it and a greedy rollout (the baseline) with the edit-distance reward of
        ``scst.edit_reward`` against the reference, and minimise L = -(1/B) sum_b (r_sample - r_greedy)_b log pi(sample_b).  The
        attention regulariser is not part of this objective.  ``train_step`` then returns the device vector [L, mean r_sample,
        mean r_greedy, mean sampled length] and ``getLoss`` -L; ``decoder.last_fed_tokens`` holds the samples ([B, L-1], the first
        token is the caption's).  tau is a device scalar, so a captured step graph picks up a new tau without re-capture.  ``None``
        or 0: back to cross-entropy.  Refused together with scheduled sampling and with data parallelism (``dist``)."""
        tau = 0.0 if temperature is None else float(temperature)
        if not (tau >= 0.0 and math.isfinite(tau)):
            raise ValueError("temperature must be a finite tau > 0, or None / 0 for cross-entropy (got %r)" % (temperature,))
        if tau > 0.0:
            if self.sampling_prob > 0.0:
                raise _lib.LatexOcrB200Error("self-critical training and scheduled sampling exclude each other: call "
                                             "set_sampling_prob(0) first")
            if self.dist is not None:
                raise _lib.LatexOcrB200Error("self-critical training is not available with data parallelism (dist)")
            if self._scst_temp_dev is None:
                self._scst_temp_dev = torch.zeros((), dtype=torch.float32, device=self.device)
                self._scst_one = torch.ones((), dtype=torch.float32, device=self.device)
            self._scst_temp_dev.fill_(tau)
        self.scst_temperature = tau

    def train_mode(self, flag=True):
        self.encoder.train(flag)
        self.decoder.train(flag)

    # --- the fused train step --------------------------------------------------------------------
    @staticmethod
    def _trainable_ranges(store, module):
        """Contiguous {offset, count} ranges of the flat store owned by parameters with requires_grad=True, or None when
        nothing is frozen."""
        frozen = {p_._lo_store_name for p_ in module.parameters() if not p_.requires_grad}
        if not frozen:
            return None
        ranges = []
        for name, (off, n, _) in sorted(store.offsets.items(), key=lambda kv: kv[1][0]):
            if name in frozen:
                continue
            if ranges and ranges[-1][0] + ranges[-1][1] == off:
                ranges[-1][1] += n
            else:
                ranges.append([off, n])
        return ranges

    def _adam(self, store, grad_scale=1.0, module=None):
        L = _lib.lib()
        ranges = self._trainable_ranges(store, module) if module is not None else None
        if ranges is None:
            check(L.lo_adam_step(ptr(store.master), ptr(store.grad), ptr(store.m), ptr(store.v), ptr(store.shadow), store.numel,
                                 ptr(store.adam_state), 0.9, 0.999, 1e-8, float(grad_scale), stream_ptr()))
            return
        # fine_tune()/fine_tune_embeddings() (seq2seq_torch.py:102-113, :246-253): torch.optim.Adam skips parameters without a
        # gradient, so frozen slices see neither moment decay nor an update
        import ctypes
        flat = [x for r in ranges for x in r]
        arr = (ctypes.c_int64 * max(len(flat), 1))(*flat)
        check(L.lo_adam_step_ranges(ptr(store.master), ptr(store.grad), ptr(store.m), ptr(store.v), ptr(store.shadow), arr, len(ranges),
                                    ptr(store.adam_state), 0.9, 0.999, 1e-8, float(grad_scale), stream_ptr()))

    def _step_body(self, img, caps, decode_lengths, dropout_mask):
        """encoder fwd -> decoder fwd + loss -> decoder bwd -> encoder bwd -> (grad all-reduce) -> Adam x2.
        img: CUDA fp32 [N,1,H,W]; caps: CUDA int64 [N,L] sorted rows.  Returns the device loss vector."""
        if self.scst_temperature > 0.0:
            return self._scst_step_body(img, caps, decode_lengths, dropout_mask)
        N = img.shape[0]
        enc_out = self.encoder.forward_raw(img, need_grad=True)
        R = enc_out.shape[1] * enc_out.shape[2]
        enc_flat = enc_out.view(N, R, enc_out.shape[3])
        ss = self._ss_prob_dev if self.sampling_prob > 0.0 else None
        ws = self.decoder.run_forward(enc_flat, caps, decode_lengths, with_loss=True, need_grad=True, dropout_mask=dropout_mask,
                                      ss_prob=ss)
        self.decoder.last_fed_tokens = ws["t"]["fed"] if ss is not None else None
        self.decoder.run_backward(ws)
        scale = 1.0
        if self.dist is not None:
            self.dist.reduce_async(self.decoder.store.grad)        # decoder bucket flies while the encoder backward runs
            scale = 1.0 / self.dist.world_size
        denc = ws["t"]["denc"].view(N, enc_out.shape[1], enc_out.shape[2], enc_out.shape[3])
        if self.dist is None:
            self.encoder.backward_raw(tuple(img.shape), denc)
        else:
            # encoder buckets: each layer's gradient is all-reduced as soon as its weight-gradient kernels are enqueued (last
            # conv first), small layers coalesced; only the first convs' few kB are left exposed before Adam
            self.encoder.backward_raw(tuple(img.shape), denc, on_layer_grad=self.dist.layer_hook(self.encoder))
            self.dist.wait()
        self._adam(self.decoder.store, scale, self.decoder)
        self._adam(self.encoder.store, scale, self.encoder)
        return ws["t"]["loss"]

    def _scst_step_body(self, img, caps, decode_lengths, dropout_mask):
        """The self-critical step (set_self_critical): encoder fwd -> sample pass (p = 1, tau, train-mode dropout) -> greedy rollout
        (p = 1, no dropout, its own workspace) -> rewards -> policy gradient -> generic decoder bwd (teacher forcing on the sample)
        -> encoder bwd -> Adam x2.  Returns the device vector [L, mean r_sample, mean r_greedy, mean n_b]."""
        from . import scst
        dec = self.decoder
        N, V = img.shape[0], dec.vocab_size
        enc_out = self.encoder.forward_raw(img, need_grad=True)
        R = enc_out.shape[1] * enc_out.shape[2]
        enc_flat = enc_out.view(N, R, enc_out.shape[3])
        T = max(decode_lengths)
        ws = dec.run_forward(enc_flat, caps, decode_lengths, with_loss=False, need_grad=True, dropout_mask=dropout_mask,
                             ss_prob=self._scst_one, ss_temp=self._scst_temp_dev)
        gw = dec.run_forward(enc_flat, caps, decode_lengths, with_loss=False, need_grad=False, ss_prob=self._scst_one,
                             key=("scst_rollout", N, T, R))
        t = ws["t"]
        if t.get("scst_dpred") is None:
            f32 = dict(dtype=torch.float32, device=self.device)
            t["scst_dpred"] = torch.zeros(N, T, V, **f32)
            t["scst_partial"] = torch.zeros(N, T, **f32)
            t["scst_stats"] = torch.zeros(4, **f32)
            t["scst_r"] = (torch.zeros(N, **f32), torch.zeros(N, **f32), torch.zeros(N, **f32),
                           torch.zeros(N, dtype=torch.int32, device=self.device))
        fed = t["fed"]
        dec.last_fed_tokens = fed
        r_s, r_g, adv, n_len = scst.rewards(fed, caps, self._end_id(), greedy=gw["t"]["fed"], out=t["scst_r"])
        scst.pg_grad(t["logits"], ws["ldl"], fed, adv, n_len, self._scst_temp_dev, N, T, V, t["scst_dpred"], t["scst_partial"],
                     t["scst_stats"], r_sample=r_s, r_greedy=r_g)
        has_do = 0 if dropout_mask is None else (2 if isinstance(dropout_mask, str) else 1)
        a = dec.fill_args(ws, enc_flat, N, T, R, has_do, ss_prob=self._scst_one)
        a.dpred_ext = t["scst_dpred"].data_ptr()       # generic mode: teacher forcing on the sampled tokens
        a.dpred_stride = V
        dec.run_backward(ws)
        denc = t["denc"].view(N, enc_out.shape[1], enc_out.shape[2], enc_out.shape[3])
        self.encoder.backward_raw(tuple(img.shape), denc)
        self._adam(self.decoder.store, 1.0, self.decoder)
        self._adam(self.encoder.store, 1.0, self.encoder)
        return t["scst_stats"]

    def _end_id(self):
        """The END id: the vocabulary's, else the last id (the default of the decode entry points)."""
        return self._vocab.id_end if self._vocab is not None else self._n_tok - 1

    def _keepalive(self):
        """Everything a captured graph replays on (the bounded workspace caches may evict their entries later)."""
        return [list(self.decoder._ws.values()), list(self.encoder._ws.values())]

    def _param_modules(self):
        """Every module with a flat parameter store that the step updates."""
        return tuple(getattr(self, n) for n in ("encoder", "decoder", "row_encoder", "layer2") if getattr(self, n, None) is not None)

    def _stores(self):
        """Every flat parameter store the step updates (snapshotted around the pre-capture warm-up steps)."""
        return tuple(m_.store for m_ in self._param_modules())

    def train_step(self, img, formula, sync=False):
        """img: float tensor [N,1,H,W] (CPU pinned or CUDA); formula: int64 [N,L] (CPU or CUDA).
        Returns the device loss vector [total, ce, reg, n_valid], or [L, mean r_sample, mean r_greedy, mean n_b] in self-critical
        mode (set_self_critical); no host sync unless sync=True."""
        N, L = formula.shape
        if self.scst_temperature > 0.0 and self.dist is not None:
            raise _lib.LatexOcrB200Error("self-critical training is not available with data parallelism (dist)")
        # the step writes the flat gradient buffers; autograd use or zero_grad(set_to_none=True) may have re-pointed p.grad
        for m_ in self._param_modules():
            bind_grads(m_, m_.store)
        lengths = torch.full((N, 1), L, dtype=torch.long)                       # img2seq_torch.py:144
        lens, sort_ind = lengths.squeeze(1).sort(dim=0, descending=True)        # seq2seq_torch.py:286 (host, tiny)
        decode_lengths = (lens - 1).tolist()
        img_d = img.to(self.device, non_blocking=True)
        caps_d = formula.to(self.device, non_blocking=True)
        if not torch.equal(sort_ind, torch.arange(N)):
            si = sort_ind.to(self.device)
            img_d, caps_d = img_d[si], caps_d[si]
        T = L - 1
        if not self.use_graph:
            mask = self.decoder.make_dropout_mask(N, T)
            loss = self._step_body(img_d if img_d.dtype == torch.uint8 else img_d.float(), caps_d, decode_lengths, mask)
        else:
            loss = self._graph_step(img_d, caps_d, decode_lengths)
        if sync:
            torch.cuda.synchronize()
        return loss

    def _graph_step(self, img_d, caps_d, decode_lengths):
        frozen = tuple(p_._lo_store_name for m_ in (self.encoder, self.decoder) for p_ in m_.parameters() if not p_.requires_grad)
        key = (tuple(img_d.shape), img_d.dtype, tuple(caps_d.shape), self.decoder.training, frozen, self.sampling_prob > 0.0,
               self.scst_temperature > 0.0)
        g = self._graphs.get(key)
        if g is None:
            N, T = caps_d.shape[0], caps_d.shape[1] - 1
            st = {"img": torch.zeros(img_d.shape, dtype=torch.uint8 if img_d.dtype == torch.uint8 else torch.float32, device=self.device),
                  "caps": torch.zeros(caps_d.shape, dtype=torch.int64, device=self.device)}
            st["img"].copy_(img_d)
            st["caps"].copy_(caps_d)
            # warm-up outside capture (allocates workspaces, sets kernel attributes); it must not train:
            # parameters, Adam moments/step and the bf16 shadows are restored afterwards
            stores = self._stores()
            snap = [{k: getattr(S, k).clone() for k in ("master", "m", "v", "adam_state", "shadow") if getattr(S, k) is not None}
                    for S in stores]
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    mask = self.decoder.make_dropout_mask(N, T)
                    self._step_body(st["img"], st["caps"], decode_lengths, mask)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            for S, sn in zip(stores, snap):
                for k, v in sn.items():
                    getattr(S, k).copy_(v)
                S.mark_shadow_current()          # the restore put the shadow back too: no re-cast inside the capture
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                mask = self.decoder.make_dropout_mask(N, T)
                st["loss"] = self._step_body(st["img"], st["caps"], decode_lengths, mask)
            st["graph"] = graph          # capture records the launches, it does not execute them
            # the graph replays on the workspaces that were live during capture: keep them alive even if the bounded
            # workspace caches evict their entries
            st["keep"] = self._keepalive()
            g = self._graphs[key] = st
        g["img"].copy_(img_d, non_blocking=True)
        g["caps"].copy_(caps_d, non_blocking=True)
        g["graph"].replay()
        return g["loss"]

    def getLoss(self, img, formula, lr=None, dropout=None, training=True):
        """img2seq_torch.py:136-172.  Returns -loss as a Python float (one device->host read)."""
        loss = self.train_step(img, formula)
        return -float(loss[0].item())

    # --- epoch loop: img2seq_torch.py:90-134 / base_torch.py:169-206 ------------------------------
    def _run_train_epoch(self, config, train_set, val_set, epoch, lr_schedule):
        from .data import minibatches, pad_batch_formulas, pad_batch_images
        batch_size = config.batch_size
        self.train_mode(True)
        losses = []
        t0 = time.time()
        nimg = 0
        if getattr(self, "_batcher", None) is None:
            from .data import PinnedBatcher
            self._batcher = PinnedBatcher(self._vocab.id_pad, self._vocab.id_end)
        for i, (img, formula) in enumerate(minibatches(train_set, batch_size)):
            # pad_batch_images (utils/image.py:27-44, 255 padding) / pad_batch_formulas (utils/text.py:141-164) straight into pinned
            # staging buffers (one per shape bucket): uint8 pixels [N,1,H,W] (img2seq_torch.py:115-117; conv1 casts on the GPU: 4x
            # less H2D, same values) and int64 ids.  getLoss synchronises on the loss, so a buffer is free again when it returns.
            img = self._batcher.images(img)
            formula = self._batcher.formulas(formula)
            loss_eval = self.getLoss(img, formula=formula, lr=getattr(lr_schedule, "lr", None),
                                     dropout=getattr(config, "dropout", None), training=True)
            losses.append(loss_eval)
            nimg += img.shape[0]
            if lr_schedule is not None:
                lr_schedule.update(batch_no=epoch * ((len(train_set) + batch_size - 1) // batch_size) + i)
        self.last_epoch_stats = {"images_per_s": nimg / max(time.time() - t0, 1e-9), "mean_neg_loss": float(np.mean(losses)) if losses else 0.0}
        score = self.last_epoch_stats["mean_neg_loss"]
        if val_set is not None and self._vocab is not None:
            scores = self.evaluate(config, val_set)                                  # img2seq_torch.py:128-132
            score = scores["perplexity"]
            self.last_epoch_stats.update(scores)
            if lr_schedule is not None:
                lr_schedule.update(score=score)
        return score

    def train(self, config, train_set, val_set, lr_schedule):
        """base_torch.py:169-206 / base.py:95-140: epoch loop, weights saved whenever the epoch score is a new best (>=), early
        stopping through ``lr_schedule.stop_training``.  Resume (base.py:40-47, :107-108): epochs below ``self.startepoch`` —
        set by ``restore_latest()`` from the newest ``model.cpkt-<epoch>`` — are skipped."""
        best_score = None
        for epoch in range(config.n_epochs):
            if epoch < getattr(self, "startepoch", 0):
                continue
            score = self._run_train_epoch(config, train_set, val_set, epoch, lr_schedule)
            if best_score is None or score >= best_score:
                best_score = score
                if self._dir_output is not None:
                    self.save_session(epoch)
            if lr_schedule is not None and getattr(lr_schedule, "stop_training", False):
                break
        return best_score

    # --- inference / evaluation: img2seq.py:198-285 (TF surface) ----------------------------------------
    def _decode_ids(self, images, start_id=None, decoding=None, beam_size=None):
        """Token ids per hypothesis rank: list[n_hyp][N] of id lists (NOT truncated), as ``pred_test.ids`` after the
        reshapes of img2seq.py:236-241 / :265-268."""
        from . import decode
        decoding = decoding or getattr(self._config, "decoding", "greedy")
        end_id = self._end_id()
        start_id = end_id - 1 if start_id is None else start_id          # default: the PAD id (no START in the torch flavour)
        L = int(getattr(self._config, "max_length_formula", 150))
        self.train_mode(False)
        br = bracket_rule(self._config, self._vocab)
        if decoding == "greedy":
            return [decode.greedy_decode(self, images, start_id, end_id, L, brackets=br).tolist()], end_id
        if decoding != "beam_search" and decoding != "beam":
            raise NotImplementedError("decoding=%r: 'greedy' or 'beam_search' (model.json:13)" % (decoding,))
        beam = int(beam_size or getattr(self._config, "beam_size", 5))
        # a bracket rule holds along lineages: with it on, the hypotheses are followed back from their final slots
        kw = {"brackets": br, "finalize": "backtrack"} if br is not None else {}
        ids, _ = decode.beam_decode(self, images, start_id, end_id, beam, L,
                                    div_gamma=float(getattr(self._config, "div_gamma", 1)),
                                    div_prob=float(getattr(self._config, "div_prob", 0)),
                                    length_penalty=getattr(self._config, "length_penalty", 0) or 0,
                                    coverage_penalty=getattr(self._config, "coverage_penalty", 0) or 0, **kw)
        return [ids[:, k].tolist() for k in range(beam)], end_id

    def predict_batch(self, images, start_id=None, decoding=None, beam_size=None):
        """img2seq.py:256-277.  images: tensor [N,1,H,W] (float or uint8) or a list of HxWx1 arrays (padded like
        ``pad_batch_images``).  Returns list[n_hyp][N]: each prediction truncated at END and, when the vocabulary has an
        ``id_to_tok`` table, joined into the formula string like the reference (token-id lists otherwise)."""
        if not torch.is_tensor(images):
            from .data import pad_batch_images
            images = torch.from_numpy(pad_batch_images(list(images))).permute(0, 3, 1, 2).contiguous()
        return self._format(*self._decode_ids(images, start_id, decoding, beam_size))

    def predict_images(self, images, start_id=None, decoding=None, beam_size=None):
        """``predict_batch`` for a list of images of different sizes ([1,H,W] tensors or HxWx1 arrays), each decoded at its own
        size in one time loop: no padding to the largest image, so an image's prediction does not depend on the other images of
        the call (``predict_batch`` keeps the reference's padding).  Same return value as ``predict_batch``."""
        return self._format(*self._decode_ids(list(images), start_id, decoding, beam_size))

    def _format(self, hyps, end_id):
        """list[n_hyp][N] of id lists -> each prediction truncated at END, joined into the formula string when the vocabulary has
        an ``id_to_tok`` table."""
        from . import decode
        rev = getattr(self._vocab, "id_to_tok", None)
        out = []
        for hyp in hyps:
            trunc = decode.truncate_end(hyp, end_id)
            out.append([" ".join(rev[i] for i in p) for p in trunc] if rev is not None else trunc)
        return out

    def predict(self, img):
        """img2seq.py:278-285: one image, one string (or id list) per hypothesis rank."""
        return [hyp[0] for hyp in self.predict_batch([img])]

    def _teacher_forced_ce(self, img, formula_t, lens, start_id):
        """(sum of CE over the real tokens incl. END, number of such tokens) of one padded batch — ``ce_words`` / ``n_words`` of
        img2seq.py:72-75 on the torch-flavour decoder (inputs prefixed with START, targets = tokens then END)."""
        inp = torch.cat([torch.full((formula_t.shape[0], 1), start_id, dtype=torch.int64), formula_t], dim=1)
        with torch.no_grad():
            enc = self.encoder(img.to(self.device))
            preds, caps, dl, _, _ = self.decoder(enc, inp.to(self.device), lens + 1)
        tgt = caps[:, 1:]
        ce_sum, n_tok = 0.0, 0
        for b, n in enumerate(dl):
            lp = torch.log_softmax(preds[b, :n].float(), dim=-1)                 # host-side metric arithmetic (plumbing)
            ce_sum += float(-lp.gather(1, tgt[b, :n].unsqueeze(1)).sum().item())
            n_tok += int(n)
        return ce_sum, n_tok

    def write_prediction(self, config, test_set, start_id=None):
        """img2seq.py:215-254: decodes the whole set, writes ``ref.txt`` / ``hyp_<i>.txt`` under ``config.dir_answers`` through
        ``write_answers`` and returns (files, perplexity) with perplexity = -exp(sum CE / n_words) (negated so that 'higher
        is better' model selection works, :252)."""
        from . import metrics
        from .data import minibatches, pad_batch_formulas, pad_batch_images
        self.train_mode(False)
        end_id, pad_id = self._vocab.id_end, self._vocab.id_pad
        start_id = pad_id if start_id is None else start_id
        refs, hyps = [], None
        ce_words, n_words = 0.0, 0
        for imgs, formulas in minibatches(test_set, config.batch_size):
            img = torch.from_numpy(pad_batch_images(imgs)).permute(0, 3, 1, 2).contiguous()
            formula, length = pad_batch_formulas(formulas, pad_id, end_id)
            ce, n = self._teacher_forced_ce(img, torch.from_numpy(formula.astype(np.int64)),
                                            torch.from_numpy(length.astype(np.int64)).unsqueeze(1), start_id)
            ce_words += ce
            n_words += n
            ids, _ = self._decode_ids(img, start_id)
            if hyps is None:
                hyps = [[] for _ in ids]
            for k, h in enumerate(ids):
                hyps[k] += h
            refs += [list(map(int, f)) for f in formulas]
        rev = getattr(self._vocab, "id_to_tok", None) or {i: str(i) for i in range(self._n_tok)}
        dir_answers = getattr(config, "dir_answers", None) or os.path.join(self._dir_output or ".", "answers") + os.sep
        files = metrics.write_answers(refs, hyps or [[]], rev, dir_answers, end_id)
        perp = -float(np.exp(ce_words / float(max(n_words, 1))))
        return files, perp

    def _run_evaluate(self, config, test_set):
        """img2seq.py:198-213: scores of hypothesis 0 against the references through the answer files."""
        from . import metrics
        files, perp = self.write_prediction(config, test_set)
        scores = metrics.score_files(files[0], files[1])
        scores["perplexity"] = perp
        return scores

    def evaluate(self, config, test_set, start_id=None):
        """base.py:142-160 with the TF path's evaluation semantics (the torch path's own evaluate is broken, SURVEY quirk
        Q6): BLEU-4 / edit distance / exact match of hypothesis 0 + negated perplexity."""
        return self._run_evaluate(config, test_set)

    # --- checkpoints: state_dict round-trips with the reference modules ----------------------------
    def state_dict(self):
        return {"encoder": self.encoder.state_dict(), "decoder": self.decoder.state_dict()}

    def load_state_dict(self, sd):
        self.encoder.load_state_dict(sd["encoder"])
        self.decoder.load_state_dict(sd["decoder"])
        self._graphs.clear()                         # captured steps hold the old bf16 shadows' VALUES only through memory

    def save(self, path=None):
        path = path or os.path.join(self._dir_output or ".", "model.pt")
        torch.save({k: {n: t.detach().cpu().contiguous() for n, t in v.items()} for k, v in self.state_dict().items()}, path)
        return path

    def restore(self, path=None, map_location=None):
        """base_torch.py:150-160 (``model_path=None`` -> the default path of ``save()``)."""
        path = path or os.path.join(self._dir_output or ".", "model.pt")
        self.load_state_dict(torch.load(path, map_location=map_location or self.device))

    def auto_restore(self):
        """base_torch.py:146-148: restore the default checkpoint if it exists."""
        path = os.path.join(self._dir_output or ".", "model.pt")
        if os.path.isfile(path):
            self.restore(path)
            return True
        return False

    # TF-style epoch checkpoints (base.py:33-69): ``<dir_output>/model_weights/model.cpkt-<epoch>``, ``max_to_keep=1``,
    # and on start-up the newest one is loaded and its epoch becomes ``startepoch``
    def _dir_model(self):
        return os.path.join(self._dir_output or ".", "model_weights")

    @staticmethod
    def _ckpt_epoch(name):
        idx = name.find("-")                         # base.py:45-46
        try:
            return int(name[idx + 1:].split(".")[0]) if idx >= 0 else None
        except ValueError:
            return None

    def save_session(self, epoch):
        """base.py:60-68 (tf.train.Saver(max_to_keep=1).save(..., global_step=epoch)): parameters AND both Adam states, so a
        resumed run continues the same optimisation."""
        d = self._dir_model()
        os.makedirs(d, exist_ok=True)
        path = os.path.join(d, "model.cpkt-%d" % epoch)
        blob = {"epoch": int(epoch), "state_dict": {k: {n: t.detach().cpu().contiguous() for n, t in v.items()}
                                                    for k, v in self.state_dict().items()}}
        opt = {}
        for name, mod in (("encoder", self.encoder), ("decoder", self.decoder)):
            S = mod.store
            if S.m is not None:
                opt[name] = {"m": S.m.cpu(), "v": S.v.cpu(), "adam_state": S.adam_state.cpu()}
        blob["optimizer"] = opt
        torch.save(blob, path + ".tmp")
        os.replace(path + ".tmp", path)
        for f in os.listdir(d):                      # max_to_keep=1
            if f.startswith("model.cpkt-") and f != os.path.basename(path) and not f.endswith(".tmp"):
                os.remove(os.path.join(d, f))
        return path

    def latest_checkpoint(self):
        d = self._dir_model()
        if not os.path.isdir(d):
            return None
        c = [(self._ckpt_epoch(f), f) for f in os.listdir(d) if f.startswith("model.cpkt-") and not f.endswith(".tmp")]
        c = [x for x in c if x[0] is not None]
        return os.path.join(d, max(c)[1]) if c else None

    def restore_latest(self):
        """base.py:40-47: load the newest epoch checkpoint, set ``startepoch`` to its epoch number (the reference re-runs
        that epoch: ``epoch < startepoch`` skips only the earlier ones).  Returns the epoch or None."""
        self.startepoch = 0
        path = self.latest_checkpoint()
        if path is None:
            return None
        blob = torch.load(path, map_location=self.device)
        self.load_state_dict(blob["state_dict"])
        for name, mod in (("encoder", self.encoder), ("decoder", self.decoder)):
            o = blob.get("optimizer", {}).get(name)
            if o is not None:
                S = mod.store
                S.ensure_adam(self.lr)
                S.m.copy_(o["m"])
                S.v.copy_(o["v"])
                S.adam_state.copy_(o["adam_state"])
        self.startepoch = int(blob["epoch"])
        return self.startepoch
