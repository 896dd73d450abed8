"""Test helpers: sampling decode (lo_sample_args) restated in float64 on the CPU oracles' own cells.

Row b of step t, logits x [V]: q = softmax(x / tau); the tokens ordered by q descending, then index ascending; top-k (k >= 1)
keeps the first k, top-p (p < 1) each token whose predecessors' mass is < p; the token is argmax over the kept v of
x_v / tau - log(-log u_v), the lowest index among equals.  A row is finished after its first END and then emits END and adds
nothing; its log-prob sums log_softmax(x)[token] (temperature 1, unfiltered) through its first END.  The loop is greedy decode's
(dynamic_decode.py:38-61): it runs until every row is finished, a row being finished also once time >= max_iter.

Cells: oracle/ref_model.py (torch flavour), oracle/ref_tf_model.py (TF flavour), tests/decoder2_decode_oracle.py (two layers),
each over enc tiled to n rows per image.  Nothing here changes the oracle package."""
import math

import numpy as np
import torch
import torch.nn.functional as F

import decoder2_decode_oracle as d2o
from oracle import ref_model as rm
from oracle import ref_tf_model as tfm


def keep_mask(x, tau, top_k, top_p):
    """(kept [V] bool, margin): the filter of one row of logits x (float64 numpy), margin = the least |mass before v - p| over
    the tokens, inf with top-p off (how far the kept set is from changing under a rounding of the masses)"""
    x = np.asarray(x, dtype=np.float64)
    V = x.shape[0]
    z = x / tau
    q = np.exp(z - z.max())
    q /= q.sum()
    order = np.lexsort((np.arange(V), -q))             # q descending, then index ascending
    before = np.concatenate(([0.0], np.cumsum(q[order])[:-1]))
    keep_pos = np.ones(V, dtype=bool)
    if top_k > 0:
        keep_pos &= np.arange(V) < top_k
    margin = math.inf
    if top_p < 1.0:
        keep_pos &= before < top_p
        margin = float(np.abs(before - top_p).min())
    kept = np.zeros(V, dtype=bool)
    kept[order[keep_pos]] = True
    return kept, margin


def draw(x, tau, kept, u):
    """argmax over the kept v of x_v / tau - log(-log u_v), the first maximum"""
    s = np.asarray(x, dtype=np.float64) / tau - np.log(-np.log(np.asarray(u, dtype=np.float64)))
    s = np.where(kept, s, -np.inf)
    return int(np.argmax(s))


def search(cell, B, end_id, max_iter, tau, top_k, top_p, u):
    """Sampling decode of B rows over ``cell(tok)`` -> logits [B, V] (tok None at time 0).  ``u`` [>= steps, B, V].  Returns
    (ids [B, steps], log-probs [B], margin: the least top-p margin of any draw)."""
    u = torch.as_tensor(u).double().numpy()
    finished = np.zeros(B, dtype=bool)
    logp = np.zeros(B)
    out, tok, time, margin = [], None, 0, math.inf
    while not finished.all():
        x = cell(tok).double()
        ls = torch.log_softmax(x, dim=-1).numpy()
        x = x.numpy()
        ids = np.full(B, end_id, dtype=np.int64)
        for b in range(B):
            if finished[b]:
                continue
            kept, m = keep_mask(x[b], tau, top_k, top_p)
            margin = min(margin, m)
            ids[b] = draw(x[b], tau, kept, u[time, b])
            logp[b] += ls[b, ids[b]]
        finished |= ids == end_id
        finished |= time >= max_iter
        out.append(ids)
        tok = torch.from_numpy(ids)
        time += 1
    return torch.from_numpy(np.stack(out, axis=1)), torch.from_numpy(logp), margin


def torch_cell(pd, enc, n, start_id):
    """the torch-flavour cell (ref_decode.cell_step) over enc [N, R, C] tiled to N * n rows"""
    rep = lambda t: t.repeat_interleave(n, dim=0)
    att1 = F.linear(enc, pd["attention.encoder_att.weight"], pd["attention.encoder_att.bias"])
    h, c = rm.init_hidden_state(pd, enc)
    st = {"enc": rep(enc), "att1": rep(att1), "h": rep(h), "c": rep(c)}
    B = st["h"].shape[0]

    def cell(tok):
        tok = torch.full((B,), start_id, dtype=torch.long) if tok is None else tok
        ctx, _ = rm.attention_forward(pd, st["enc"], st["h"], st["att1"])
        gate = torch.sigmoid(F.linear(st["h"], pd["f_beta.weight"], pd["f_beta.bias"]))
        x = torch.cat([F.embedding(tok, pd["embedding.weight"]), gate * ctx], dim=1)
        st["h"], st["c"] = rm.lstm_cell(pd, x, st["h"], st["c"])
        return F.linear(st["h"], pd["fc.weight"], pd["fc.bias"])
    return cell, B


def tf_cell(p, enc, n):
    """the Genthial cell (ref_tf_model.cell_step) over enc [N, R, C] tiled to N * n rows, the start token at time 0"""
    rep = lambda t: t.repeat_interleave(n, dim=0)
    att_img = enc @ p["att_img.kernel"]
    c, h, o = tfm.initial_state(p, enc)
    st = {"enc": rep(enc), "att": rep(att_img), "s": (rep(c), rep(h), rep(o))}
    B = st["enc"].shape[0]

    def cell(tok):
        emb = p["start_token"].expand(B, -1) if tok is None else F.embedding(tok, p["embedding_table"])
        logits, st["s"], _ = tfm.cell_step(p, st["enc"], st["att"], emb, *st["s"])
        return logits
    return cell, B


def decoder2_cell(pd, p2, enc, n, start_id):
    """the two-layer cell of decoder2_decode_oracle over enc tiled to N * n rows"""
    step, _, st = d2o.cell(pd, p2, enc, n, start_id)
    return (lambda tok: step(tok)[0]), st["h"].shape[0]
