"""Test helpers: the beam search of the CPU oracles with the length and coverage penalties of lo_beam_penalty.

The loop is the reference's beam cell as oracle/ref_decode.py and oracle/ref_tf_model.py restate it (beam_search_decoder_cell.py:
98-187: log-softmax, finished rows masked to [END: 0, else: dtype.min], only beam 0 at time 0, the diversity penalty of :258-287,
top-k over beam x V with the lower index first among equals, state gather by parents), and the oracles' own cells step it.  What
it adds is the ranking of GNMT (Wu et al. 2016, eq. 14) in the form of TF's BeamSearchDecoder(length_penalty_weight=alpha):

    new_len = len[k] + (finished[k] or v == END ? 0 : 1)
    cov'    = finished[k] ? cov[k] : cov[k] + alpha_t[k]
    score   = carried / LP[new_len] + beta * sum_r ln(min(max(cov'_r, 1e-30), 1)),   LP[l] = ((5 + l) / 6) ** alpha

with a finished row's non-END candidates at dtype.min.  The top-k ranks by score, each winner carries its raw `carried` as its
log-prob, and its length and coverage follow it.  LP is computed in float64 and rounded once to the dtype of the search, as the
library's caller does.  With alpha = beta = 0 the search is the oracles' own, bit for bit."""
import torch
import torch.nn.functional as F

from oracle import ref_decode as rd
from oracle import ref_model as rm
from oracle import ref_tf_model as tfm


def length_penalty_table(alpha, n, dtype=torch.float32):
    """LP[l] = ((5 + l) / 6) ** alpha for l = 0..n-1 (GNMT eq. 14; TF beam_search_decoder._length_penalty)"""
    return (((5.0 + torch.arange(n, dtype=torch.float64)) / 6.0) ** float(alpha)).to(dtype)


def search(cell, reorder, N, beam, V, end_id, max_iter, alpha=0.0, beta=0.0, div_gamma=1.0, div_prob=0.0, div_u=None,
           dtype=torch.float32):
    """The penalised beam search over a cell.  ``cell(tok)`` steps the N*beam rows (tok: the previous ids [N*beam], None at time 0)
    and returns (logits [N*beam, V], attention weights [N*beam, R]); ``reorder(rows)`` gathers the cell state by rows.  Returns
    ids and parents [N, steps, beam], the log-probs [N, beam] and the scores [N, beam] of the final slots."""
    pen = alpha != 0 or beta > 0
    LP = length_penalty_table(alpha, max_iter + 2, dtype)
    fmin = torch.finfo(dtype).min
    log_probs = torch.zeros(N, beam, dtype=dtype)
    scores = log_probs
    finished = torch.zeros(N, beam, dtype=torch.bool)
    length = torch.zeros(N, beam, dtype=torch.long)
    cov = None
    not_end = torch.arange(V) != end_id
    ids_t, parents_t = [], []
    tok, time = None, 0
    while not bool(finished.all()):                                                   # dynamic_decode.py:38-40
        logits, a = cell(tok)
        step_lp = torch.log_softmax(logits.view(N, beam, V), dim=-1)                   # :146
        fin_row = torch.full((V,), fmin, dtype=dtype)
        fin_row[end_id] = 0.0
        f = finished.unsqueeze(-1).to(dtype)
        step_lp = (1.0 - f) * step_lp + f * fin_row                                    # mask_probs :353-367
        total = log_probs.unsqueeze(-1) + step_lp                                      # :150
        if div_u is not None:
            total = rd.add_div_penalty(total, div_gamma, div_prob, div_u[time].view(N, beam, V))   # :151-152
        new_len = length.unsqueeze(-1) + ((~finished).unsqueeze(-1) & not_end).long()
        score = total
        if pen:
            if alpha != 0:
                score = score / LP[new_len]
            if beta > 0:
                al = a.view(N, beam, -1).to(dtype)
                prev = cov if cov is not None else torch.zeros_like(al)
                cov = torch.where(finished.unsqueeze(-1), prev, prev + al)
                term = beta * torch.log(cov.clamp(1e-30, 1.0)).sum(dim=-1)
                score = score + term.unsqueeze(-1)
            score = torch.where(finished.unsqueeze(-1) & not_end, torch.tensor(fmin, dtype=dtype), score)
        flat = score[:, 0] if time == 0 else score.reshape(N, beam * V)                # :156-160
        vals, idx = rd._topk_low_index_first(flat, beam)                               # :161
        new_ids, new_parents = idx % V, idx // V                                       # :164-165
        carried = total[:, 0] if time == 0 else total.reshape(N, beam * V)
        log_probs = torch.gather(carried, 1, idx)
        lens = new_len[:, 0] if time == 0 else new_len.reshape(N, beam * V)
        length = torch.gather(lens, 1, idx)
        if cov is not None:
            cov = cov[torch.arange(N).unsqueeze(1), new_parents]
        scores = vals
        finished = torch.gather(finished, 1, new_parents) | (new_ids == end_id)      # :171-174
        reorder((new_parents + torch.arange(N).unsqueeze(1) * beam).view(-1))           # gather_helper :370-391
        ids_t.append(new_ids)
        parents_t.append(new_parents)
        finished = finished | torch.tensor(time >= max_iter)                           # dynamic_decode.py:49-51
        tok = new_ids.view(-1)
        time += 1
    return torch.stack(ids_t, dim=1), torch.stack(parents_t, dim=1), log_probs, scores


def _finish(out, finalize):
    ids, parents, log_probs, scores = out
    return (ids if finalize == "reference" else rd.backtrack(ids, parents)), log_probs, scores


def beam_decode(p, enc, start_id, end_id, beam, max_iter, finalize="reference", alpha=0.0, beta=0.0, div_gamma=1.0, div_prob=0.0,
                div_u=None):
    """ref_decode.beam_decode with the penalties: the torch-flavour cell (ref_decode.cell_step, its attention weights kept).
    Returns ids [N, steps, beam], log-probs [N, beam], scores [N, beam]."""
    N = enc.shape[0]
    V = p["fc.weight"].shape[0]
    att1 = F.linear(enc, p["attention.encoder_att.weight"], p["attention.encoder_att.bias"])
    h, c = rm.init_hidden_state(p, enc)
    st = {"enc": enc.repeat_interleave(beam, dim=0), "att1": att1.repeat_interleave(beam, dim=0),     # tile_beam :332-350
          "h": h.repeat_interleave(beam, dim=0), "c": c.repeat_interleave(beam, dim=0)}

    def cell(tok):
        tok = torch.full((N * beam,), start_id, dtype=torch.long) if tok is None else tok
        ctx, a = rm.attention_forward(p, st["enc"], st["h"], st["att1"])
        gate = torch.sigmoid(F.linear(st["h"], p["f_beta.weight"], p["f_beta.bias"]))
        x = torch.cat([F.embedding(tok, p["embedding.weight"]), gate * ctx], dim=1)
        st["h"], st["c"] = rm.lstm_cell(p, x, st["h"], st["c"])
        return F.linear(st["h"], p["fc.weight"], p["fc.bias"]), a

    def reorder(rows):
        st["h"], st["c"] = st["h"][rows], st["c"][rows]

    out = search(cell, reorder, N, beam, V, end_id, max_iter, alpha, beta, div_gamma, div_prob, div_u, enc.dtype)
    return _finish(out, finalize)


def tf_beam_decode(p, enc, end_id, beam, max_iter, finalize="reference", alpha=0.0, beta=0.0, div_gamma=1.0, div_prob=0.0,
                   div_u=None):
    """ref_tf_model.beam_decode with the penalties, on the Genthial cell (ref_tf_model.cell_step).  Returns ids [N, steps, beam],
    log-probs [N, beam], scores [N, beam]."""
    N = enc.shape[0]
    V = p["y_W_o"].shape[1]
    att_img = enc @ p["att_img.kernel"]
    c, h, o = tfm.initial_state(p, enc)
    rep = lambda x: x.repeat_interleave(beam, dim=0)                                   # tile_beam :332-350
    st = {"enc": rep(enc), "att": rep(att_img), "s": (rep(c), rep(h), rep(o))}

    def cell(tok):
        emb = p["start_token"].expand(N * beam, -1) if tok is None else F.embedding(tok, p["embedding_table"])
        logits, st["s"], a = tfm.cell_step(p, st["enc"], st["att"], emb, *st["s"])
        return logits, a

    def reorder(rows):
        st["s"] = tuple(x[rows] for x in st["s"])

    out = search(cell, reorder, N, beam, V, end_id, max_iter, alpha, beta, div_gamma, div_prob, div_u, enc.dtype)
    return _finish(out, finalize)
