"""TensorFlow-flavour ``Img2SeqModel`` — the surface of model/img2seq.py on the sm_90a kernels: ``build_train`` /
``build_pred``, ``_run_train(config, train_set, val_set, epoch, lr_schedule)`` (:144-196), ``write_prediction`` /
``_run_evaluate`` semantics (:198-254, perplexity negated like :252), ``predict_batch(images)`` / ``predict(img)`` (:256-285).

Encoder: the same 6-conv stack as the torch flavour with the TF input normalisation (img - 128) / 128 fused into conv1
(model/encoder.py:26-27; SAME/VALID paddings and SAME pools coincide with the torch stack for even sizes, SURVEY §8-A.1).
Decoder: ``tf_decoder.Decoder`` (Genthial cell).  Loss: masked CE (img2seq.py:68-71).  Optimiser: Adam on the two flat stores
(tf.train.AdamOptimizer, :104; epsilon 1e-8 like the torch flavour), optional clip_by_global_norm (:116-121).
"""
import ctypes
import math
import os
import time

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr, stream_ptr
from .data import minibatches, pad_batch_formulas, pad_batch_images
from .encoder import EncoderCNN
from .params import bind_grads
from .tf_decoder import Decoder, TfDecArgs


class _Cfg:
    """config view that adds input_norm='tf' without mutating the caller's object"""

    def __init__(self, base):
        self._base = base
        self.input_norm = "tf"

    def __getattr__(self, k):
        return getattr(self._base, k)


class Img2SeqModel:
    def __init__(self, config, dir_output=None, vocab=None, device=None, precision=None, impl=None):
        self._config = config
        self._dir_output = dir_output
        self._vocab = vocab
        self.device = torch.device(device or getattr(config, "device", "cuda"))
        if self.device.type != "cuda":
            raise _lib.LatexOcrB200Error("latex_ocr_b200 runs on CUDA devices only (no CPU fallback)")
        self.precision = precision or getattr(config, "precision", "bf16")
        self.impl = impl if impl is not None else getattr(config, "conv_impl", "tc" if self.precision == "bf16" else "simt")
        self.encoder = self.decoder = None
        self.lr = None
        self.dist = None          # set by latex_ocr_b200.dist.attach(model): data-parallel gradient all-reduce
        self.last_epoch_stats = {}
        self.sampling_prob = 0.0          # scheduled sampling in the train step (set_sampling_prob)
        self.scst_temperature = 0.0       # self-critical training (set_self_critical); 0: cross-entropy
        self.set_sampling_prob(getattr(config, "sampling_prob", 0.0) or 0.0)

    # img2seq.py:33-53 / :55-66: the TF graph is replaced by the two modules
    def build_train(self, config=None):
        config = config or self._config
        self._build()
        method = str(getattr(config, "lr_method", "adam")).lower()
        # img2seq.py:98-111: adam | adagrad | sgd | rmsprop, TF 1.12 update rules (csrc/lo_optim.cu:tf_optim_kernel)
        kinds = {"adam": 1, "sgd": 2, "adagrad": 3, "rmsprop": 4}
        if method not in kinds:
            raise NotImplementedError("Unknown method {}".format(method))          # img2seq.py:111
        self.lr_method, self._opt_kind = method, kinds[method]
        self.clip = float(getattr(config, "clip", -1))
        self.set_lr(float(getattr(config, "lr_init", 1e-3)))
        return self

    def build_pred(self, config=None):
        self._build()
        return self

    def _build(self):
        if self.encoder is None:
            self.encoder = EncoderCNN(_Cfg(self._config), device=self.device, precision=self.precision, impl=self.impl)
            self.decoder = Decoder(self._config, self._vocab.n_tok, self._vocab.id_end, device=self.device, precision=self.precision,
                                   impl=self.impl)

    def set_lr(self, lr):
        self.lr = float(lr)
        kind = getattr(self, "_opt_kind", 1)
        for m in (self.encoder, self.decoder):
            S = m.store
            fresh = S.m is None
            S.ensure_adam(lr)                     # slot buffers m (s1) / v (s2) + the device {step, lr} pair
            if fresh and kind == 3:
                S.m.fill_(0.1)                    # tf.train.AdagradOptimizer: initial_accumulator_value = 0.1
            elif fresh and kind == 4:
                S.m.fill_(1.0)                    # tf.train.RMSPropOptimizer: the rms slot starts at ones
            S.set_lr(lr)

    def set_sampling_prob(self, p):
        """Scheduled sampling (Bengio et al. 2015) in ``compute_gradients`` / ``train_step`` / ``_run_train``: from the next step on,
        the decoder step after step t consumes the model's own argmax of step t's logits with probability p instead of
        ``formula[:, t]`` (tf_decoder.Decoder.train_outputs documents the rule).  The loss stays the masked CE against the formula,
        so data parallelism works unchanged.  No schedule is built in: set p per epoch.  0 runs the teacher-forced step."""
        p = float(p)
        if not 0.0 <= p <= 1.0:
            raise ValueError("sampling_prob must lie in [0, 1] (got %r)" % (p,))
        if p > 0.0 and self.scst_temperature > 0.0:
            raise _lib.LatexOcrB200Error("scheduled sampling and self-critical training exclude each other: call "
                                         "set_self_critical(None) first")
        self.sampling_prob = p

    def set_self_critical(self, temperature):
        """Self-critical sequence training (SCST; Rennie et al. 2017) in ``train_step`` / ``_run_train``.  ``temperature`` = tau > 0:
        from the next step on, a step samples one formula per image from softmax(logits / tau) inside the CUDA time loop (with the
        step's dropout), scores it and a greedy rollout (the baseline, lo_tfdec_greedy) with the edit-distance reward of
        ``scst.rewards`` against the formula, and minimises L = -(1/N) sum_b (r_sample - r_greedy)_b log pi(sample_b), then applies
        the configured optimiser (with ``clip``).  ``train_step`` then returns the device vector [L, mean r_sample, mean r_greedy,
        mean sampled length], and ``decoder.last_fed_tokens`` holds the samples [N, T].  ``None`` or 0: back to cross-entropy.
        Refused together with scheduled sampling and with data parallelism (``dist``)."""
        tau = 0.0 if temperature is None else float(temperature)
        if not (tau >= 0.0 and math.isfinite(tau)):
            raise ValueError("temperature must be a finite tau > 0, or None / 0 for cross-entropy (got %r)" % (temperature,))
        if tau > 0.0:
            if self.sampling_prob > 0.0:
                raise _lib.LatexOcrB200Error("self-critical training and scheduled sampling exclude each other: call "
                                             "set_sampling_prob(0) first")
            if self.dist is not None:
                raise _lib.LatexOcrB200Error("self-critical training is not available with data parallelism (dist)")
        self.scst_temperature = tau

    # ---------------------------------------------------------------------------------------------
    def _to_device_images(self, images):
        """list of HWC uint8 arrays (or an [N,H,W,1] array) -> CUDA uint8 [N,1,H,W] (pad_batch_images: 255 padding)."""
        if isinstance(images, torch.Tensor):
            img = images
        else:
            img = torch.from_numpy(pad_batch_images(images))
        if img.dim() == 4 and img.shape[-1] == 1:
            img = img.permute(0, 3, 1, 2)
        return img.contiguous().to(self.device, non_blocking=True)

    def compute_gradients(self, images, formulas, dropout=1.0):
        """Forward + loss + backward (+ the data-parallel all-reduce): images as above, formulas = list of id lists (padded here like
        _get_feed_dict img2seq.py:132-135) or an (int array [N,T], lengths [N]) pair.  Gradients land in the two flat stores;
        returns the device loss vector [mean CE, mean CE, 0, n_words]."""
        img, formula_t, length_t, keep_h, keep_o = self._step_inputs(images, formulas, dropout)
        N = img.shape[0]
        enc = self.encoder.forward_raw(img, need_grad=True)
        n_words = None
        if self.dist is not None and self.dist.world_size > 1:
            # the loss is a mean over valid tokens: all-reduce the token count (one scalar, SURVEY §8-e), then the SUM of the rank
            # gradients is the gradient of the global mean
            import torch.distributed as tdist
            nw = torch.tensor([float(length_t.sum())], device=self.device)
            tdist.all_reduce(nw, group=self.dist.group)
            n_words = float(nw.item())
        loss, denc = self.decoder.loss_and_backward(enc, formula_t, length_t, keep_h, keep_o, n_words, self.sampling_prob)
        if self.dist is not None:
            self.dist.reduce_async(self.decoder.store.grad)             # flies while the encoder backward runs
        self.encoder.backward_raw(tuple(img.shape), denc.view(N, enc.shape[1], enc.shape[2], enc.shape[3]))
        if self.dist is not None:
            self.dist.reduce_async(self.encoder.store.grad)
            self.dist.wait()
        return loss

    def _step_inputs(self, images, formulas, dropout):
        """(images on the device, formula int64 [N,T] on the device, lengths int32 [N], keep_h, keep_o) of one train step; binds the
        flat gradient buffers, which the step writes (autograd use or zero_grad(set_to_none=True) may have re-pointed p.grad)."""
        if isinstance(formulas, tuple):
            formula, length = formulas
        else:
            formula, length = pad_batch_formulas(formulas, self._vocab.id_pad, self._vocab.id_end)
        formula_t = torch.as_tensor(np.asarray(formula), dtype=torch.int64).to(self.device, non_blocking=True)
        length_t = torch.as_tensor(np.asarray(length), dtype=torch.int32)
        img = self._to_device_images(images)
        N = img.shape[0]
        for m_ in (self.encoder, self.decoder):
            bind_grads(m_, m_.store)
        keep_h = keep_o = None
        if dropout is not None and float(dropout) < 1.0:
            kp, T = float(dropout), formula_t.shape[1]
            keep_h = (torch.rand(N, T, self.decoder.D, device=self.device) < kp).float() / kp
            keep_o = (torch.rand(N, T, self.decoder.O, device=self.device) < kp).float() / kp
        return img, formula_t, length_t, keep_h, keep_o

    def _scst_gradients(self, images, formulas, dropout):
        """The self-critical gradients (set_self_critical): encoder fwd -> sample pass (p = 1, tau, the step's keep masks) ->
        greedy rollout (lo_tfdec_greedy for T steps in the decode workspace) -> rewards -> policy gradient into d logits -> generic
        decoder bwd (teacher forcing on the sample) -> encoder bwd.  Returns the device vector [L, mean r_sample, mean r_greedy,
        mean n_b]."""
        from . import scst
        img, formula_t, _, keep_h, keep_o = self._step_inputs(images, formulas, dropout)
        dec = self.decoder
        N, T = formula_t.shape
        V, end = dec.V, self._vocab.id_end
        enc = self.encoder.forward_raw(img, need_grad=True)
        one, tau = dec.sampling_scalars(1.0, self.scst_temperature)
        ws = dec.run_forward(enc, formula_t, None, keep_h, keep_o, ss_prob=one, ss_temp=tau)
        fed = dec.last_fed_tokens = ws["fed"]
        L, gws, ga = dec._args(ws["enc"], N, T, ws["enc"].shape[1], decode=True)
        gws["enc"] = ws["enc"]
        if gws.get("rollout") is None:
            gws["rollout"] = torch.zeros(N, T, dtype=torch.int64, device=self.device)
        check(L.lo_tfdec_greedy(ctypes.byref(ga), end, T, gws["rollout"].data_ptr(), None, stream_ptr()))
        if ws.get("scst") is None:
            f32 = dict(dtype=torch.float32, device=self.device)
            ws["scst"] = {"dlogits": torch.zeros(N, T, V, **f32), "partial": torch.zeros(N, T, **f32), "stats": torch.zeros(4, **f32),
                          "r": (torch.zeros(N, **f32), torch.zeros(N, **f32), torch.zeros(N, **f32),
                                torch.zeros(N, dtype=torch.int32, device=self.device))}
        sc = ws["scst"]
        r_s, r_g, adv, n_len = scst.rewards(fed, formula_t, end, greedy=gws["rollout"], out=sc["r"], layout="tf")
        scst.pg_grad_tf(ws["logits"], fed, adv, n_len, tau, sc["dlogits"], sc["partial"], sc["stats"], r_sample=r_s, r_greedy=r_g)
        a = TfDecArgs.from_buffer_copy(ws["args"])
        a.dlogits_ext, a.dlogits_stride = sc["dlogits"].data_ptr(), V      # generic mode: teacher forcing on the sample
        check(L.lo_tfdec_backward(ctypes.byref(a), stream_ptr()))
        self.encoder.backward_raw(tuple(img.shape), ws["denc"].view(N, enc.shape[1], enc.shape[2], enc.shape[3]))
        return sc["stats"]

    def apply_gradients(self):
        """optimizer.apply_gradients (img2seq.py:113-123): optional clip_by_global_norm, then Adam on both stores."""
        L = _lib.lib()
        scale = 1.0
        if self.clip > 0:                                                   # tf.clip_by_global_norm (img2seq.py:116-121)
            gn = float(torch.sqrt(self.encoder.store.grad.pow(2).sum() + self.decoder.store.grad.pow(2).sum()))
            scale = min(1.0, self.clip / max(gn, 1e-30))
        kind = getattr(self, "_opt_kind", 1)
        # TF defaults: Adam beta1 0.9, beta2 0.999, epsilon 1e-8 (outside the bias correction); RMSProp decay 0.9, epsilon 1e-10
        b1, b2, eps = (0.9, 0.9, 1e-10) if kind == 4 else (0.9, 0.999, 1e-8)
        for m in (self.decoder, self.encoder):
            S = m.store
            check(L.lo_tf_optim_step(kind, ptr(S.master), ptr(S.grad), ptr(S.m), ptr(S.v), ptr(S.shadow), S.numel, ptr(S.adam_state), b1, b2, eps,
                     float(scale), stream_ptr()))

    def train_step(self, images, formulas, dropout=1.0):
        """One update (img2seq.py:163-170).  Returns the device loss vector [mean CE, mean CE, 0, n_words], or [L, mean r_sample,
        mean r_greedy, mean n_b] in self-critical mode (set_self_critical)."""
        if self.scst_temperature > 0.0:
            if self.dist is not None:
                raise _lib.LatexOcrB200Error("self-critical training is not available with data parallelism (dist)")
            loss = self._scst_gradients(images, formulas, dropout)
        else:
            loss = self.compute_gradients(images, formulas, dropout)
        self.apply_gradients()
        return loss

    def _run_train(self, config, train_set, val_set, epoch, lr_schedule):
        """img2seq.py:144-196.  In self-critical mode the epoch statistics are the means of the steps' [L, r_sample, r_greedy,
        n_b] instead of the CE perplexity, and without ``val_set`` the score is the mean greedy reward (higher is better)."""
        batch_size = config.batch_size
        nbatches = (len(train_set) + batch_size - 1) // batch_size
        scst = self.scst_temperature > 0.0
        t0, n_img, losses = time.time(), 0, []
        for i, (img, formula) in enumerate(minibatches(train_set, batch_size)):
            if lr_schedule is not None:
                self.set_lr(lr_schedule.lr)
            loss = self.train_step(img, formula, dropout=getattr(config, "dropout", 1.0))
            losses.append(loss.clone() if scst else loss[0:1].clone())
            n_img += len(img)
            if lr_schedule is not None:
                lr_schedule.update(batch_no=epoch * nbatches + i)
        torch.cuda.synchronize()
        images_per_s = n_img / max(time.time() - t0, 1e-9)
        if scst:
            m = torch.stack(losses).mean(dim=0).tolist() if losses else [float("nan")] * 4
            self.last_epoch_stats = {"scst_loss": m[0], "reward_sample": m[1], "reward_greedy": m[2], "sample_length": m[3],
                                     "images_per_s": images_per_s}
            if val_set is None:
                return m[2]
        else:
            mean_loss = float(torch.cat(losses).mean()) if losses else float("nan")
            self.last_epoch_stats = {"loss": mean_loss, "perplexity_train": float(np.exp(mean_loss)), "images_per_s": images_per_s}
            if val_set is None:
                return -float(np.exp(mean_loss))
        scores = self.evaluate(config, val_set)
        self.last_epoch_stats.update(scores)
        if lr_schedule is not None:
            lr_schedule.update(score=scores["perplexity"])
        return scores["perplexity"]

    def evaluate(self, config, test_set):
        """_run_evaluate / write_prediction (img2seq.py:198-254): perplexity = -exp(sum CE / n_words) from the teacher-forced
        pass with dropout off, text metrics of hypothesis 0 of the decoded ids."""
        from . import decode, metrics
        refs, hyps = [], []
        ce_words, n_words = 0.0, 0.0
        for imgs, formulas in minibatches(test_set, config.batch_size):
            img = self._to_device_images(imgs)
            formula, length = pad_batch_formulas(formulas, self._vocab.id_pad, self._vocab.id_end)
            enc = self.encoder.forward_raw(img)
            ws = self.decoder.run_forward(enc, torch.as_tensor(formula.astype(np.int64)).to(self.device),
                                          torch.as_tensor(length.astype(np.int32)))
            l = ws["loss"].tolist()
            ce_words += l[0] * l[3]
            n_words += l[3]
            ids = self.decoder.decode(enc, **self._decode_kw()).ids
            hyp0 = ids if ids.dim() == 2 else ids[:, :, 0]
            hyps += decode.truncate_end(hyp0.tolist(), self._vocab.id_end)
            refs += [list(map(int, f)) for f in formulas]
        scores = metrics.score(refs, hyps)
        scores["perplexity"] = -float(np.exp(ce_words / max(n_words, 1.0)))
        return scores

    def predict_batch(self, images):
        """img2seq.py:256-275: list over hypotheses (1 for greedy, beam_size for beam search) of N token-id lists, truncated at END."""
        enc = self.encoder.forward_raw(self._to_device_images(images))
        return self._format(self.decoder.decode(enc, **self._decode_kw()).ids)

    def _decode_kw(self):
        """The decode keywords of ``config.balanced_brackets``: none when off; else the LaTeX bracket rule of the vocabulary and
        lineage-consistent beam hypotheses (the rule holds along lineages)."""
        from .img2seq import bracket_rule
        br = bracket_rule(self._config, self._vocab)
        return {} if br is None else {"brackets": br, "finalize": "backtrack"}

    def predict_images(self, images):
        """``predict_batch`` for a list of images of different sizes (HxWx1 uint8 arrays or [1,H,W] tensors), each decoded at its
        own size in one time loop: no padding to the largest image, so an image's prediction does not depend on the other images
        of the call (``predict_batch`` keeps the reference's padding).  The images are sorted by shape and the encoder runs once
        per shape.  A list of more than ``tf_decoder.MAX_ROWS`` decoder rows (images x beam) is decoded in consecutive chunks of
        input order, each chunk as its own call.  Same return value as ``predict_batch``."""
        from .tf_decoder import MAX_ROWS
        images = list(images)
        if not images:
            raise ValueError("no images")
        per = max(1, MAX_ROWS // self.decoder._tiles)
        hyps = None
        for k in range(0, len(images), per):
            part = self._predict_chunk(images[k:k + per])
            hyps = part if hyps is None else [h + p for h, p in zip(hyps, part)]
        return hyps

    def _predict_chunk(self, images):
        from . import decode
        dec = self.decoder
        lay = decode.ragged_layout(images, self.encoder.out_hw)
        steps = dec.max_length_formula + 2
        ws = dec.packed_workspace(lay.counts, steps)               # decode order: sorted by shape
        decode.encode_packed(self.encoder, lay, ws["enc"], self.device)
        ids = dec.decode_packed(ws, steps, **self._decode_kw()).ids
        return self._format(ids[decode._inverse(lay.order).to(ids.device)])

    def _format(self, ids):
        """greedy ids [N, time] or beam ids [N, time, beam] -> list over hypotheses of N token-id lists, truncated at END"""
        from . import decode
        if ids.dim() == 2:
            return [decode.truncate_end(ids.tolist(), self._vocab.id_end)]
        return [decode.truncate_end(ids[:, :, k].tolist(), self._vocab.id_end) for k in range(ids.shape[2])]

    def predict(self, img):
        return [h[0] for h in self.predict_batch([img])]

    # checkpoints
    def state_dict(self):
        return {"encoder": self.encoder.state_dict(), "decoder": self.decoder.state_dict()}

    def load_state_dict(self, sd):
        self.encoder.load_state_dict(sd["encoder"])
        self.decoder.load_state_dict(sd["decoder"])

    def save(self, path=None):
        path = path or os.path.join(self._dir_output or ".", "model_tf.pt")
        torch.save({k: {n: t.detach().cpu().contiguous() for n, t in v.items()} for k, v in self.state_dict().items()}, path)
        return path

    def restore(self, path):
        self.load_state_dict(torch.load(path, map_location=self.device))
