"""Test helpers: the bracket rule of lo_bracket_rule on the CPU oracles' own cells.

Each decode row keeps a stack of kinds.  Before step t's token choice the stack takes the row's token of step t-1 (a push for an
opening token, a pop for a closing one) unless the row was already finished, and every token the row may not take gets logit -inf:
with d the depth and r = max_steps - 1 - t the steps left, a close of kind k needs d > 0 and k on top, an open d < max_depth and
d + 1 <= r, a neutral token d <= r, END d == 0.  Beam search gathers the stacks by parent rows with the cell state.  The wrappers
below apply that to the cells of oracle/ref_decode.py (torch flavour), oracle/ref_tf_model.py (TF flavour) and
tests/decoder2_decode_oracle.py (two layers), and run them through the oracles' own searches: greedy decode as
ref_decode.greedy_decode, tests/beam_penalty_oracle.search and tests/sample_oracle.search.  In beam search a finished row's
logits are left unmasked: its log-probs are replaced by the finished mask anyway, and -inf there would turn that mask into NaN.
Nothing here changes the oracle modules."""
import torch
import torch.nn.functional as F

import beam_penalty_oracle as bpo
import decoder2_decode_oracle as d2o
import sample_oracle as so
from oracle import ref_model as rm
from oracle import ref_tf_model as tfm


class Stacks:
    """the rule's per-row state over B rows of a call of ``max_steps`` steps"""

    def __init__(self, rule, B, end_id, max_steps, mask_finished=True):
        self.role, self.max_depth, self.end_id, self.max_steps = rule.role, rule.max_depth, end_id, max_steps
        self.mask_finished = mask_finished
        self.stack = [[] for _ in range(B)]
        self.fin = [False] * B
        self.t = 0

    def allowed(self, b):
        d, r = len(self.stack[b]), self.max_steps - 1 - self.t
        top = self.stack[b][-1] if d else 0
        out = []
        for v, ro in enumerate(self.role):
            if ro < 0:
                out.append(d > 0 and top == -ro)
            elif ro > 0:
                out.append(d < self.max_depth and d + 1 <= r)
            else:
                out.append(d == 0 if v == self.end_id else d <= r)
        return torch.tensor(out)

    def step(self, logits, tok):
        """the stacks take ``tok`` (the previous ids, None at step 0), then the excluded logits of ``logits`` [B, V] become -inf"""
        if tok is not None:
            for b, v in enumerate(tok.tolist()):
                if not self.fin[b]:
                    ro = self.role[v]
                    if ro > 0:
                        self.stack[b].append(ro)
                    elif ro < 0:
                        self.stack[b].pop()
                self.fin[b] = self.fin[b] or v == self.end_id
        out = logits.clone()
        for b in range(out.shape[0]):
            if self.fin[b] and not self.mask_finished:
                continue
            out[b][~self.allowed(b)] = float("-inf")
        self.t += 1
        return out

    def reorder(self, rows):
        rows = rows.tolist()
        self.stack = [list(self.stack[r]) for r in rows]
        self.fin = [self.fin[r] for r in rows]


def masked(cell, stacks):
    """cell(tok) -> logits or (logits, attention), with the rule applied to the logits"""
    def step(tok):
        out = cell(tok)
        if isinstance(out, tuple):
            return (stacks.step(out[0], tok),) + tuple(out[1:])
        return stacks.step(out, tok)
    return step


def greedy(cell, B, rule, end_id, max_iter):
    """ref_decode.greedy_decode's loop (dynamic_decode.py:38-61) over ``cell`` under the rule: ids [B, steps]"""
    step = masked(cell, Stacks(rule, B, end_id, max_iter + 1))
    finished = torch.zeros(B, dtype=torch.bool)
    out, tok, time = [], None, 0
    while not bool(finished.all()):
        ids = torch.argmax(step(tok), dim=-1)                   # the lowest index among equal maxima
        out.append(ids)
        finished = finished | (ids == end_id) | torch.tensor(time >= max_iter)
        tok, time = ids, time + 1
    return torch.stack(out, dim=1)


def sample(cell, B, rule, end_id, max_iter, tau, top_k, top_p, u):
    """sample_oracle.search over ``cell`` under the rule: (ids [B, steps], log-probs [B], top-p margin)"""
    return so.search(masked(cell, Stacks(rule, B, end_id, max_iter + 1)), B, end_id, max_iter, tau, top_k, top_p, u)


def beam(cell, reorder, N, beam_size, V, rule, end_id, max_iter, finalize="backtrack", dtype=torch.float64, **kw):
    """beam_penalty_oracle.search over ``cell`` / ``reorder`` under the rule: (ids [N, steps, beam], log-probs, scores)"""
    st = Stacks(rule, N * beam_size, end_id, max_iter + 1, mask_finished=False)

    def reorder2(rows):
        st.reorder(rows)
        reorder(rows)
    out = bpo.search(masked(cell, st), reorder2, N, beam_size, V, end_id, max_iter, dtype=dtype, **kw)
    return bpo._finish(out, finalize)


# ------------------------------------------------------------------------------------------------ the flavours' cells
def torch_cells(pd, enc, rows_per_img, start_id):
    """(cell, reorder) of the torch flavour (ref_decode.cell_step, its attention kept) over enc [N,R,C] tiled to N * rows_per_img"""
    rep = lambda x: x.repeat_interleave(rows_per_img, dim=0)
    att1 = F.linear(enc, pd["attention.encoder_att.weight"], pd["attention.encoder_att.bias"])
    h, c = rm.init_hidden_state(pd, enc)
    st = {"enc": rep(enc), "att1": rep(att1), "h": rep(h), "c": rep(c)}
    B = st["h"].shape[0]

    def cell(tok):
        tok = torch.full((B,), start_id, dtype=torch.long) if tok is None else tok
        ctx, a = rm.attention_forward(pd, st["enc"], st["h"], st["att1"])
        gate = torch.sigmoid(F.linear(st["h"], pd["f_beta.weight"], pd["f_beta.bias"]))
        x = torch.cat([F.embedding(tok, pd["embedding.weight"]), gate * ctx], dim=1)
        st["h"], st["c"] = rm.lstm_cell(pd, x, st["h"], st["c"])
        return F.linear(st["h"], pd["fc.weight"], pd["fc.bias"]), a

    def reorder(rows):
        st["h"], st["c"] = st["h"][rows], st["c"][rows]
    return cell, reorder


def tf_cells(p, enc, rows_per_img):
    """(cell, reorder) of the Genthial cell (ref_tf_model.cell_step) over enc tiled to N * rows_per_img, the start token at time 0"""
    rep = lambda x: x.repeat_interleave(rows_per_img, dim=0)
    att_img = enc @ p["att_img.kernel"]
    c, h, o = tfm.initial_state(p, enc)
    st = {"enc": rep(enc), "att": rep(att_img), "s": (rep(c), rep(h), rep(o))}
    B = st["enc"].shape[0]

    def cell(tok):
        emb = p["start_token"].expand(B, -1) if tok is None else F.embedding(tok, p["embedding_table"])
        logits, st["s"], a = tfm.cell_step(p, st["enc"], st["att"], emb, *st["s"])
        return logits, a

    def reorder(rows):
        st["s"] = tuple(x[rows] for x in st["s"])
    return cell, reorder


def decoder2_cells(pd, p2, enc, rows_per_img, start_id):
    """(cell, reorder) of the two-layer cell of decoder2_decode_oracle"""
    step, reorder, _ = d2o.cell(pd, p2, enc, rows_per_img, start_id)
    return step, reorder


def first(cell):
    """a cell returning (logits, attention) as one returning logits"""
    return lambda tok: cell(tok)[0]

