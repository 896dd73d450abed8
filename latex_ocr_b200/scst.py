"""Self-critical sequence training (SCST; Rennie et al., CVPR 2017, applied to this model by Wang & Liu, IJDAR 2021) on both
decoder flavours: the sequence reward and the policy gradient on the device (csrc/lo_scst.cu).

The reward of a hypothesis h against its reference is the per-row form of ``metrics.edit_distance``: both are truncated at the
first END (``metrics.truncate_end``) and r(h) = 1 - lev(h, ref) / max(|h|, |ref|), 1 when both are empty.  The fused train step
(``Img2SeqModel.set_self_critical``) uses these kernels; the autograd route needs only ``edit_reward``:

    with torch.no_grad():                            # the baseline: a greedy rollout (eval mode: no dropout)
        dec.eval(); dec(enc, caps, lens, sampling_prob=1.0); greedy = dec.last_fed_tokens; dec.train()
    preds, caps_s, dl, _, _ = dec(enc, caps, lens, sampling_prob=1.0, sampling_temperature=tau)   # the sample
    adv = edit_reward(dec.last_fed_tokens, caps_s, end_id) - edit_reward(greedy, caps_s, end_id)

The rollout runs first because a later forward of the same shape overwrites the state the sample's backward needs.

The TensorFlow flavour (``tf_decoder.Decoder``) draws every token, the first one included: its samples are
``last_fed_tokens`` [N, T] in the layout of ``formula``, and ``layout="tf"`` selects its step convention (``rewards``) and its
time-major logits (``pg_grad_tf``).  Its autograd route:

    with torch.no_grad():                            # the baseline: greedy decode for T steps, no dropout
        greedy = dec.decode(enc, max_steps=T).ids
    logits, alphas = dec.train_outputs(enc, formula, sampling_prob=1.0, sampling_temperature=tau)      # the sample
    fed = dec.last_fed_tokens
    r_s, r_g, adv, n_len = rewards(fed, formula, end_id, greedy=greedy, layout="tf")
    lp = torch.log_softmax(logits / tau, -1).gather(2, fed[:, :, None])[:, :, 0]                       # log pi(fed[b][t])
    steps = torch.arange(T, device=lp.device)[None, :] < n_len[:, None]                              # t < n_b
    (-(adv[:, None] * lp * steps).sum() / N).backward()
"""
import torch

from . import _lib
from ._lib import check, ptr, stream_ptr


def _i64(t):
    t = t.to(dtype=torch.int64)
    return t if t.stride(-1) == 1 else t.contiguous()


def rewards(hyp, ref, end_id, greedy=None, out=None, layout="torch"):
    """One launch of lo_scst_edit_reward.  hyp [B, Lh], ref [B, Lr], greedy (optional) [B, Lg]: CUDA integer tensors.
    Returns (r_sample, r_greedy, adv, n_len): fp32 [B] each (r_greedy and adv None without ``greedy``) and int32 [B] n_len, the
    number of sampled steps the policy gradient differentiates.  ``layout="torch"``: hyp[b][0] is the given start token, and n_len is
    the first t >= 1 with hyp[b][t] == end_id, else Lh - 1.  ``layout="tf"`` (tf_decoder.Decoder, lo_scst_edit_reward_tf): every
    token was drawn, and n_len = min(e + 1, Lh) for the first e >= 0 with hyp[b][e] == end_id, else Lh.  The rewards are the same in
    both.  ``out``: those four tensors to write into (a captured step reuses them)."""
    if layout not in ("torch", "tf"):
        raise ValueError("layout must be 'torch' or 'tf' (got %r)" % (layout,))
    hyp, ref = _i64(hyp), _i64(ref)
    B = hyp.shape[0]
    if ref.shape[0] != B or (greedy is not None and greedy.shape[0] != B):
        raise ValueError("hypotheses and references need the same number of rows")
    if out is None:
        r_s = torch.empty(B, dtype=torch.float32, device=hyp.device)
        out = (r_s, torch.empty_like(r_s), torch.empty_like(r_s), torch.empty(B, dtype=torch.int32, device=hyp.device))
    r_s, r_g, adv, n_len = out
    Lg, gs = 0, 0
    if greedy is None:
        r_g = adv = None
    else:
        greedy = _i64(greedy)
        Lg, gs = greedy.shape[1], greedy.stride(0)
    fn = _lib.lib().lo_scst_edit_reward if layout == "torch" else _lib.lib().lo_scst_edit_reward_tf
    check(fn(ptr(hyp), hyp.stride(0), hyp.shape[1], ptr(greedy), gs, Lg, ptr(ref), ref.stride(0), ref.shape[1], B, int(end_id), ptr(r_s), ptr(r_g), ptr(adv), ptr(n_len), stream_ptr()))
    return r_s, r_g, adv, n_len


def edit_reward(hyp, ref, end_id):
    """Per-row edit-distance reward of the hypotheses ``hyp`` [B, Lh] against ``ref`` [B, Lr] (CUDA integer tensors), both
    truncated at the first ``end_id``: fp32 [B] on the device, exact (integer distances)."""
    return rewards(hyp, ref, end_id)[0]


def pg_grad(preds, pred_stride, fed, adv, n_len, temp, B, T, V, dpred, partial, stats, r_sample=None, r_greedy=None):
    """One lo_scst_pg_grad: d L / d preds into ``dpred`` [B, T, V] and {L, mean r_sample, mean r_greedy, mean n_len} into
    ``stats`` [4] for L = -(1/B) sum_b adv_b sum_{t=1..n_b} log softmax(preds[b][t-1] / tau)[fed[b][t]] (``temp``: a CUDA scalar
    tau).  ``preds``: fp32 rows (b, t) ``pred_stride`` apart; ``fed`` int64 [B, >= T]; ``partial`` fp32 [B, T] scratch."""
    check(_lib.lib().lo_scst_pg_grad(ptr(preds), int(pred_stride), ptr(fed), fed.stride(0), ptr(adv), ptr(n_len), ptr(temp),
                                     ptr(r_sample), ptr(r_greedy), B, T, V, ptr(dpred), dpred.stride(-2), ptr(partial), ptr(stats),
                                     stream_ptr()))


def pg_grad_tf(logits, fed, adv, n_len, temp, dlogits, partial, stats, r_sample=None, r_greedy=None):
    """One lo_scst_pg_grad_tf over the time-major logits of tf_decoder.Decoder (``logits`` fp32 [T, B, ldl], its workspace layout):
    d L / d logits into ``dlogits`` [B, T, V] (batch-major, the layout of the generic backward's d logits) and {L, mean r_sample,
    mean r_greedy, mean n_len} into ``stats`` [4] for L = -(1/B) sum_b adv_b sum_{t < n_b} log softmax(logits[t][b] / tau)[fed[b][t]]
    (``temp``: a CUDA scalar tau; ``n_len`` from ``rewards(..., layout="tf")``).  ``fed`` int64 [B, >= T]; ``partial`` fp32 [B, T]
    scratch."""
    T, B, ldl = logits.shape
    V = dlogits.shape[-1]
    if logits.stride(-1) != 1 or logits.stride(1) != ldl or logits.stride(0) != B * ldl:
        raise ValueError("logits must be a contiguous [T, B, ldl] tensor")
    check(_lib.lib().lo_scst_pg_grad_tf(ptr(logits), ldl, ptr(fed), fed.stride(0), ptr(adv), ptr(n_len), ptr(temp), ptr(r_sample),
                                        ptr(r_greedy), B, T, V, ptr(dlogits), dlogits.stride(-2), ptr(partial), ptr(stats),
                                        stream_ptr()))
