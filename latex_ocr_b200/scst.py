"""Self-critical sequence training (SCST; Rennie et al., CVPR 2017, applied to this model by Wang & Liu, IJDAR 2021) on the
torch-flavour decoder: the sequence reward and the policy gradient on the device (csrc/lo_scst.cu).

The reward of a hypothesis h against its reference is the per-row form of ``metrics.edit_distance``: both are truncated at the
first END (``metrics.truncate_end``) and r(h) = 1 - lev(h, ref) / max(|h|, |ref|), 1 when both are empty.  The fused train step
(``Img2SeqModel.set_self_critical``) uses these kernels; the autograd route needs only ``edit_reward``:

    with torch.no_grad():                            # the baseline: a greedy rollout (eval mode: no dropout)
        dec.eval(); dec(enc, caps, lens, sampling_prob=1.0); greedy = dec.last_fed_tokens; dec.train()
    preds, caps_s, dl, _, _ = dec(enc, caps, lens, sampling_prob=1.0, sampling_temperature=tau)   # the sample
    adv = edit_reward(dec.last_fed_tokens, caps_s, end_id) - edit_reward(greedy, caps_s, end_id)

The rollout runs first because a later forward of the same shape overwrites the state the sample's backward needs.
"""
import torch

from . import _lib
from ._lib import check, ptr, stream_ptr


def _i64(t):
    t = t.to(dtype=torch.int64)
    return t if t.stride(-1) == 1 else t.contiguous()


def rewards(hyp, ref, end_id, greedy=None, out=None):
    """One launch of lo_scst_edit_reward.  hyp [B, Lh], ref [B, Lr], greedy (optional) [B, Lg]: CUDA integer tensors.
    Returns (r_sample, r_greedy, adv, n_len): fp32 [B] each (r_greedy and adv None without ``greedy``) and int32 [B] n_len, the
    first t >= 1 with hyp[b][t] == end_id, else Lh - 1.  ``out``: those four tensors to write into (a captured step reuses them)."""
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
    check(_lib.lib().lo_scst_edit_reward(ptr(hyp), hyp.stride(0), hyp.shape[1], ptr(greedy), gs, Lg, ptr(ref), ref.stride(0),
                                         ref.shape[1], B, int(end_id), ptr(r_s), ptr(r_g), ptr(adv), ptr(n_len), stream_ptr()))
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
