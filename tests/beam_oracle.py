"""Test helpers: what the CPU oracles' beam search computes on the way, and the attention weights of its hypotheses.

``recorded_beam`` runs ref_decode.beam_decode or ref_tf_model.beam_decode unchanged and records, by wrapping the oracle functions
that compute them for the duration of the call, every row's attention weights at every step (ref_model.attention_forward,
ref_tf_model.attention_context) and every step's top-k picks (ref_decode._topk_low_index_first), whose flat index over beam x V
gives the parents.  ``hypothesis_attention`` applies the rule of lo_beam_backtrack to that record; ``teacher_forced_attention`` /
``tf_teacher_forced_attention`` compute what a teacher-forced pass over a hypothesis's own tokens attends to."""
import contextlib

import torch

from oracle import ref_decode as rd
from oracle import ref_model as rm
from oracle import ref_tf_model as tfm


@contextlib.contextmanager
def _wrapped(module, name, record):
    fn = getattr(module, name)

    def wrapper(*args, **kw):
        out = fn(*args, **kw)
        record.append(out)
        return out
    setattr(module, name, wrapper)
    try:
        yield
    finally:
        setattr(module, name, fn)


def recorded_beam(flavour, p, enc, V, *args, **kw):
    """``flavour`` 'torch' (ref_decode.beam_decode(p, enc, *args, **kw)) or 'tf' (ref_tf_model.beam_decode); V: the vocabulary
    size.  Returns the oracle's own return value followed by alphas [N*beam, steps, R] (row i*beam + s: slot s of image i, before
    the step's top-k) and parents [N, steps, beam]."""
    N = enc.shape[0]
    att, topk = [], []
    module, name = (rm, "attention_forward") if flavour == "torch" else (tfm, "attention_context")
    with _wrapped(module, name, att), _wrapped(rd, "_topk_low_index_first", topk):
        out = (rd.beam_decode if flavour == "torch" else tfm.beam_decode)(p, enc, *args, **kw)
    assert len(att) == len(topk) == out[0].shape[1]          # one attention call and one top-k per step
    alphas = torch.stack([a for _, a in att], dim=1)
    parents = torch.stack([idx // V for _, idx in topk], dim=1)
    assert alphas.shape[0] == parents.shape[0] * parents.shape[2] == N * parents.shape[2]
    return tuple(out) + (alphas, parents)


def hypothesis_attention(alphas, parents, finalize):
    """The attention weights of the hypotheses, [N, beam, steps, R], from recorded_beam's alphas [N*beam, steps, R] and parents
    [N, steps, beam].  'reference': slot s's own rows.  'backtrack': walking back from the final slot s, the row of step t is the
    parent p of the slot the hypothesis holds at t (the row whose attention chose that token); then that slot becomes p."""
    N, S, beam = parents.shape
    al = alphas.reshape(N, beam, S, -1)
    if finalize == "reference":
        return al.clone()
    out = torch.empty_like(al)
    cur = torch.arange(beam).unsqueeze(0).repeat(N, 1)
    img = torch.arange(N).unsqueeze(1)
    for t in range(S - 1, -1, -1):
        cur = torch.gather(parents[:, t], 1, cur)
        out[:, :, t] = al[img, cur, t]
    return out


def teacher_forced_attention(p, enc, start_id, hyps):
    """Torch flavour: the attention weights of a teacher-forced pass (ref_model.decoder_forward) over each hypothesis: enc [N,R,C],
    hyps [N, beam, n] -> [N, beam, n, R]; step t is fed start_id, then hyps[..., t-1]."""
    N, beam, n = hyps.shape
    caps = torch.cat([torch.full((N * beam, 1), start_id, dtype=torch.long), hyps.reshape(N * beam, n)], dim=1)
    lens = torch.full((N * beam, 1), n + 1, dtype=torch.long)
    _, _, _, al, sort_ind = rm.decoder_forward(p, enc.repeat_interleave(beam, dim=0), caps, lens)
    out = torch.empty_like(al)
    out[sort_ind] = al
    return out.reshape(N, beam, n, -1)


def tf_teacher_forced_attention(p, enc, hyps):
    """TensorFlow flavour: the same through ref_tf_model.decoder_train_logits (step t is fed the start token, then
    hyps[..., t-1])."""
    N, beam, n = hyps.shape
    _, al = tfm.decoder_train_logits(p, enc.repeat_interleave(beam, dim=0), hyps.reshape(N * beam, n))
    return al.reshape(N, beam, n, -1)
