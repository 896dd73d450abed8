"""Test helpers: greedy and beam decode of the two-layer decoder (the EXTENSION of oracle/ref_ext.py) on the CPU.

The cell is decoder2_forward's step without dropout: layer 1 = the attention LSTM of oracle/ref_model.py started from
init_hidden_state(enc), layer 2 = nn.LSTMCell(D, D) over h1_t from a zero state, logits_t = fc(h2_t).  Greedy decode follows
oracle/ref_decode.greedy_decode line by line (start id supplied by the caller, rows keep decoding after END, at most max_iter + 1
steps); beam search is tests/beam_penalty_oracle.search over this cell, so the diversity, length and coverage penalties and both
finalize modes come with it.  Nothing here changes the oracle package."""
import torch
import torch.nn.functional as F

import beam_penalty_oracle as bpo
from oracle import ref_ext as rx
from oracle import ref_model as rm


def encode(pe, prow, img):
    """CNN -> row encoder: img [N,1,H,W] -> enc [N, R, 512]"""
    enc = rx.row_encoder_forward(prow, rm.encoder_forward(pe, img))
    return enc.reshape(enc.shape[0], -1, enc.shape[3])


def layer2_step(p2, x, h2, c2):
    """nn.LSTMCell(D, D) as ref_ext.decoder2_forward computes it"""
    g = F.linear(x, p2["cell.weight_ih"], p2["cell.bias_ih"]) + F.linear(h2, p2["cell.weight_hh"], p2["cell.bias_hh"])
    i, f, gg, o = g.chunk(4, dim=1)
    c2 = torch.sigmoid(f) * c2 + torch.sigmoid(i) * torch.tanh(gg)
    return torch.sigmoid(o) * torch.tanh(c2), c2


def cell(pd, p2, enc, rows_per_img, start_id):
    """(cell, reorder, state) over enc [N,R,C] tiled to N * rows_per_img rows, for beam_penalty_oracle.search: ``cell(tok)`` (tok
    None at time 0: the start id) steps both layers and returns (logits, attention weights of layer 1); ``reorder(rows)`` gathers
    h1, c1, h2, c2 by rows."""
    rep = lambda x: x.repeat_interleave(rows_per_img, dim=0)
    att1 = F.linear(enc, pd["attention.encoder_att.weight"], pd["attention.encoder_att.bias"])
    h, c = rm.init_hidden_state(pd, enc)
    st = {"enc": rep(enc), "att1": rep(att1), "h": rep(h), "c": rep(c)}
    st["h2"] = torch.zeros_like(st["h"])
    st["c2"] = torch.zeros_like(st["c"])
    B = st["h"].shape[0]

    def step(tok):
        tok = torch.full((B,), start_id, dtype=torch.long) if tok is None else tok
        ctx, a = rm.attention_forward(pd, st["enc"], st["h"], st["att1"])
        gate = torch.sigmoid(F.linear(st["h"], pd["f_beta.weight"], pd["f_beta.bias"]))
        x = torch.cat([F.embedding(tok, pd["embedding.weight"]), gate * ctx], dim=1)
        st["h"], st["c"] = rm.lstm_cell(pd, x, st["h"], st["c"])
        st["h2"], st["c2"] = layer2_step(p2, st["h"], st["h2"], st["c2"])
        return F.linear(st["h2"], pd["fc.weight"], pd["fc.bias"]), a

    def reorder(rows):
        for k in ("h", "c", "h2", "c2"):
            st[k] = st[k][rows]

    return step, reorder, st


def greedy_decode(pd, p2, enc, start_id, end_id, max_iter):
    """ref_decode.greedy_decode on the two-layer cell.  Returns ids [N, steps], logits [N, steps, V], attention [N, steps, R]."""
    N = enc.shape[0]
    step, _, _ = cell(pd, p2, enc, 1, start_id)
    finished = torch.zeros(N, dtype=torch.bool)
    out, logits, att = [], [], []
    tok, time = None, 0
    while not bool(finished.all()):                          # dynamic_decode.py:38-40
        lg, a = step(tok)
        ids = torch.argmax(lg, dim=-1)                       # greedy_decoder_cell.py:58 (lowest index on ties)
        out.append(ids)
        logits.append(lg)
        att.append(a)
        finished = finished | (ids == end_id)                # :62
        finished = finished | torch.tensor(time >= max_iter) # dynamic_decode.py:49-51
        tok = ids
        time += 1
    return torch.stack(out, dim=1), torch.stack(logits, dim=1), torch.stack(att, dim=1)


def beam_decode(pd, p2, enc, start_id, end_id, beam, max_iter, finalize="reference", alpha=0.0, beta=0.0, div_gamma=1.0,
                div_prob=0.0, div_u=None):
    """beam_penalty_oracle.beam_decode on the two-layer cell: ids [N, steps, beam] (the lineage under 'backtrack'), log-probs
    [N, beam], scores [N, beam]."""
    step, reorder, _ = cell(pd, p2, enc, beam, start_id)
    out = bpo.search(step, reorder, enc.shape[0], beam, pd["fc.weight"].shape[0], end_id, max_iter, alpha, beta, div_gamma, div_prob,
                     div_u, enc.dtype)
    return bpo._finish(out, finalize)
