"""CPU (-m "not gpu"): tests/decode_step_ref.py, the float64 decode step that tests/test_gpu_decode_steps.py checks the library
against, chained over whole decodes, reproduces the CPU oracles: oracle/ref_decode.py greedy and beam search,
tests/beam_penalty_oracle.py with the length and coverage penalties and the diversity penalty, tests/sample_oracle.py, and
tests/decoder2_decode_oracle.py — the same ids, and log-probs and scores within 1e-12.

The step before the choice is built from the flavours' own float64 step pieces (tests/decoder_step_ref.py, tests/tfdec_step_ref.py,
tests/lstmseq_step_ref.py) with decode's row-to-image map: rows_per_img rows per image, ragged lists of images (each image over
its own regions, its state from its own region mean).  An image of a ragged list must decode as it does alone."""
import math

import pytest
import torch

import beam_penalty_oracle as bpo
import decode_step_ref as dr
import decoder_step_ref as ds
import lstmseq_step_ref as lr
import sample_oracle as so
import tfdec_step_ref as ts

V = 30
START, END = V - 2, 5
MAX_ITER = 7


def _torch_params(seed):
    from oracle import ref_model as rm
    _, pd = rm.init_params(V, seed=seed, dtype=torch.float64)
    g = torch.Generator().manual_seed(seed)
    pd["fc.weight"] = ((torch.rand(V, 512, generator=g) * 2 - 1) * 0.5).double()
    pd["embedding.weight"] = ((torch.rand(V, 512, generator=g) * 2 - 1) * 1.0).double()
    return pd


def _tf_params(seed):
    from oracle import ref_tf_model as tfm
    p = tfm.init_params_tf(V, seed=seed, dtype=torch.float64)
    p["y_W_o"] = p["y_W_o"] * 4.0
    return p


def _layer2_params(seed):
    from oracle import ref_ext as rx
    return rx.init_params_ext(seed=seed, dtype=torch.float64)[1]


def _encs(counts, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.relu(torch.randn(n, 512, generator=g)) * 0.7).double() for n in counts]


class _Rows:
    """the decode state of B = N * rpi rows over images ``encs`` (a list of [R_i][C]): row b reads image b // rpi"""

    def __init__(self, encs, rpi):
        self.encs, self.rpi = encs, rpi
        self.counts = [e.shape[0] for e in encs]
        self.B = len(encs) * rpi
        self.mean = dr.rows_of(dr.region_means(torch.cat(encs), self.counts)[0], rpi)

    def attend(self, fn):
        """fn(image, rows) -> (alpha [n][R_i], ...): per image over its own rows; alpha padded to the largest R with zeros"""
        Rm = max(self.counts)
        al, rest = [], []
        for i in range(len(self.encs)):
            a, *o = fn(i, slice(i * self.rpi, (i + 1) * self.rpi))
            al.append(torch.nn.functional.pad(a, (0, Rm - a.shape[1])))
            rest.append(o)
        return torch.cat(al), [torch.cat(x) for x in zip(*rest)]


def torch_flavour(pd, encs, rpi, layer2=None):
    """(cell, reorder, B) of the torch flavour (DecoderWithAttention) on decoder_step_ref's pieces; with ``layer2`` the two-layer
    decoder, layer 2 on lstmseq_step_ref's cell.  cell(tok) -> (logits [B][V], alphas [B][R_max])"""
    rows = _Rows(encs, rpi)
    C = encs[0].shape[1]
    A = pd["attention.decoder_att.weight"].shape[0]
    att1 = [ds.linear(e, pd["attention.encoder_att.weight"], pd["attention.encoder_att.bias"])[0] for e in encs]
    ptab = ds.proj_table(pd, C)
    wf = pd["attention.full_att.weight"].reshape(-1)
    h, c = ds.init_state(pd, rows.mean)
    st = {"h": h, "c": c, "h2": torch.zeros_like(h), "c2": torch.zeros_like(c)}

    def cell(tok):
        tok = torch.full((rows.B,), START, dtype=torch.long) if tok is None else tok
        out1 = ds.project(pd, st["h"])
        att2, gate, hh = out1[:, :A], torch.sigmoid(out1[:, A:A + C]), out1[:, A + C:]

        def one(i, r):
            n = r.stop - r.start
            _, al, _, gctx = ds.attention(att1[i].expand(n, -1, -1), encs[i].expand(n, -1, -1), att2[r], wf, gate[r])
            return al, gctx
        al, (gctx,) = rows.attend(one)
        *_, st["c"], st["h"] = ds.cell(pd, gctx, ptab[tok], hh, st["c"])
        top = st["h"]
        if layer2 is not None:
            pre = lr.input_projection(st["h"], layer2["cell.weight_ih"], layer2["cell.bias_ih"], layer2["cell.bias_hh"])[0]
            pre = pre + lr.recurrent(st["h2"], layer2["cell.weight_hh"])[0]
            *_, st["c2"], st["h2"] = lr.cell_forward(pre, st["c2"])
            top = st["h2"]
        return ds.head(pd, top), al

    def reorder(r):
        for k in st:
            st[k] = st[k][r]
    return cell, reorder, rows.B


def tf_flavour(p, encs, rpi):
    """(cell, reorder, B) of the TF flavour on tfdec_step_ref's pieces: step 0 feeds row V of the token table (the start token)"""
    rows = _Rows(encs, rpi)
    D = p["lstm.kernel"].shape[1] // 4
    A = p["att_h.kernel"].shape[1]
    att_img = [e @ p["att_img.kernel"] for e in encs]
    table = ts.token_table(p)
    _, s = ts.initial_state(p, rows.mean)
    st = {"c": s[:, :D], "h": s[:, D:2 * D], "o": s[:, 2 * D:]}

    def cell(tok):
        row = torch.full((rows.B,), V, dtype=torch.long) if tok is None else tok
        _, st["c"], st["h"] = ts.lstm_pointwise(ts.gates_z(p, st["o"], st["h"]) + table[row], st["c"])
        out2 = ts.project_h(p, st["h"])

        def one(i, r):
            n = r.stop - r.start
            _, al, ctx = ts.attention(att_img[i].expand(n, -1, -1), encs[i].expand(n, -1, -1), out2[r, :A], p["att_beta"])
            return al, ctx
        al, (ctx,) = rows.attend(one)
        st["o"] = ts.output(p, ctx, out2[:, A:])
        return ts.logits(p, st["o"]), al

    def reorder(r):
        for k in st:
            st[k] = st[k][r]
    return cell, reorder, rows.B


# ---------------------------------------------------------------------------------------------------------------------------------
# the loops, on decode_step_ref's choices
# ---------------------------------------------------------------------------------------------------------------------------------
def greedy_loop(cell, B):
    fin = torch.zeros(B, dtype=torch.bool)
    out, tok, t = [], None, 0
    while not bool(fin.all()):
        tok, fin = dr.greedy(cell(tok)[0], fin, END)
        out.append(tok)
        fin = fin | (t >= MAX_ITER)
        t += 1
    return torch.stack(out, 1)


def sample_loop(cell, B, tau, top_k, top_p, u):
    fin = torch.zeros(B, dtype=torch.bool)
    logp = torch.zeros(B, dtype=torch.float64)
    out, tok, t = [], None, 0
    while not bool(fin.all()):
        tok, logp, fin, _ = dr.sample(cell(tok)[0], fin, logp, tau, top_k, top_p, u[t], END)
        out.append(tok)
        fin = fin | (t >= MAX_ITER)
        t += 1
    return torch.stack(out, 1), logp


def beam_loop(cell, reorder, B, beam, counts, alpha=0.0, beta=0.0, gamma=1.0, prob=0.0, div_u=None):
    """the beam search of beam_loop (csrc/lo_decoder.cu) on decode_step_ref's beam_step and coverage; returns ids, parents
    [N][steps][beam], logp and scores [N][beam]"""
    N = B // beam
    fin = torch.zeros(B, dtype=torch.bool)
    logp = torch.zeros(B, dtype=torch.float64)
    pen = alpha != 0 or beta > 0
    LP = bpo.length_penalty_table(alpha, MAX_ITER + 2, torch.float64) if alpha != 0 else None
    lens = torch.zeros(B, dtype=torch.long)
    cov, parent_rows = None, None
    ids_t, par_t, tok, t = [], [], None, 0
    while not bool(fin.all()):
        logits, al = cell(tok)
        term = None
        if beta > 0:
            cov, term, _ = dr.coverage(al, cov, parent_rows, fin, counts, beam, t, beta)
        on = gamma != 1.0 and prob != 0.0
        o = dr.beam_step(logits, logp, fin, t, beam, END, math.log(gamma) if on else 0.0, prob if on else 0.0,
                         div_u[t] if on else None, LP, term, lens if pen else None)
        logp, parent_rows, tok = o["logp"], o["parent_rows"], o["next_tok"]
        if pen:
            lens = o["len_out"]
        reorder(parent_rows)
        ids_t.append(o["ids"])
        par_t.append(o["parents"])
        fin = o["fin"].reshape(-1) | (t >= MAX_ITER)
        t += 1
    return torch.stack(ids_t, 1), torch.stack(par_t, 1), logp.view(N, beam), o["scores"].view(N, beam)


def _close(a, b):
    assert a.shape == b.shape and float((a.double() - b.double()).abs().max()) <= 1e-12, (a, b)


# ---------------------------------------------------------------------------------------------------------------------------------
# greedy
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flavour", ["torch", "tf", "two_layer"])
def test_greedy_is_the_oracle(flavour):
    from oracle import ref_decode as rd
    from oracle import ref_tf_model as tfm
    import decoder2_decode_oracle as d2o
    counts = [12, 5, 12, 31]                                       # a ragged list; each image as decoded alone
    encs = _encs(counts, 1)
    if flavour == "tf":
        p = _tf_params(2)
        got = greedy_loop(*tf_flavour(p, encs, 1)[::2])
        want = [tfm.greedy_decode(p, e[None], END, MAX_ITER)[0] for e in encs]
    elif flavour == "torch":
        p = _torch_params(2)
        got = greedy_loop(*torch_flavour(p, encs, 1)[::2])
        want = [rd.greedy_decode(p, e[None], START, END, MAX_ITER)[0] for e in encs]
    else:
        p, p2 = _torch_params(2), _layer2_params(3)
        got = greedy_loop(*torch_flavour(p, encs, 1, p2)[::2])
        want = [d2o.greedy_decode(p, p2, e[None], START, END, MAX_ITER)[0][0] for e in encs]
    for i, w in enumerate(want):
        # the batch runs until every row has finished: a row keeps its argmax after its END (the caller truncates)
        assert torch.equal(got[i, :len(w)], w), (i, got[i], w)
    assert len(set(tuple(g.tolist()) for g in got)) > 1


def test_greedy_ties_go_to_the_lowest_index():
    x = torch.tensor([[0.0, 2.0, 2.0, 1.0], [3.0, 3.0, 3.0, 3.0], [-1.0, -2.0, -1.0, -0.5]], dtype=torch.float64)
    tok, fin = dr.greedy(x, torch.tensor([False, True, False]), 2)
    assert tok.tolist() == [1, 0, 3] and fin.tolist() == [False, True, False]


# ---------------------------------------------------------------------------------------------------------------------------------
# beam search
# ---------------------------------------------------------------------------------------------------------------------------------
_BEAM = [
    # (beam, alpha, beta, diversity)
    (1, 0.0, 0.0, False),
    (3, 0.0, 0.0, False),
    (3, 0.0, 0.0, True),
    (3, 0.8, 0.0, False),
    (3, 0.0, 0.4, False),
    (5, 0.6, 0.3, True),
    (16, 0.6, 0.3, False),
]


@pytest.mark.parametrize("flavour", ["torch", "tf", "two_layer"])
@pytest.mark.parametrize("beam,alpha,beta,div", _BEAM, ids=["b%d-a%g-c%g-%s" % (b, a, c, "div" if d else "nodiv")
                                                            for b, a, c, d in _BEAM])
def test_beam_is_the_oracle(flavour, beam, alpha, beta, div):
    from oracle import ref_decode as rd
    import decoder2_decode_oracle as d2o
    N, R = 2, 12
    encs = _encs([R] * N, 4)
    enc = torch.stack(encs)
    kw = dict(alpha=alpha, beta=beta)
    if div:
        kw.update(div_gamma=0.5, div_prob=0.7,
                  div_u=torch.rand(MAX_ITER + 2, N * beam, V, generator=torch.Generator().manual_seed(5), dtype=torch.float64))
    mine = dict(alpha=alpha, beta=beta, gamma=kw.get("div_gamma", 1.0), prob=kw.get("div_prob", 0.0), div_u=kw.get("div_u"))
    if flavour == "tf":
        p = _tf_params(6)
        cell, reorder, B = tf_flavour(p, encs, beam)
        want = bpo.tf_beam_decode(p, enc, END, beam, MAX_ITER, **kw)
    elif flavour == "torch":
        p = _torch_params(3)
        cell, reorder, B = torch_flavour(p, encs, beam)
        want = bpo.beam_decode(p, enc, START, END, beam, MAX_ITER, **kw)
        if alpha == 0 and beta == 0:
            w2 = rd.beam_decode(p, enc, START, END, beam, MAX_ITER, div_gamma=kw.get("div_gamma", 1.0),
                                div_prob=kw.get("div_prob", 0.0), div_u=kw.get("div_u"))
            assert torch.equal(w2[0], want[0]) and torch.equal(w2[1], want[1])
    else:
        p, p2 = _torch_params(3), _layer2_params(4)
        cell, reorder, B = torch_flavour(p, encs, beam, p2)
        want = d2o.beam_decode(p, p2, enc, START, END, beam, MAX_ITER, **kw)
    ids, parents, logp, scores = beam_loop(cell, reorder, B, beam, [R] * N, **mine)
    assert torch.equal(ids, want[0]), (ids, want[0])
    _close(logp, want[1])
    _close(scores, want[2])


def test_beam_on_a_ragged_list_is_each_image_alone():
    """rows_per_img = beam over images of 31, 7 and 20 regions: every image's hypotheses, log-probs and scores are those of its
    own search (the coverage over its own regions)"""
    counts = [31, 7, 20]
    beam = 4
    encs = _encs(counts, 8)
    p = _torch_params(9)
    cell, reorder, B = torch_flavour(p, encs, beam)
    ids, _, logp, scores = beam_loop(cell, reorder, B, beam, counts, alpha=0.6, beta=0.3)
    for i, e in enumerate(encs):
        w_ids, w_lp, w_sc = bpo.beam_decode(p, e[None], START, END, beam, MAX_ITER, alpha=0.6, beta=0.3)
        n = w_ids.shape[1]
        assert torch.equal(ids[i, :n], w_ids[0])
        _close(logp[i], w_lp[0])
        _close(scores[i], w_sc[0])


def test_beam_step_rules():
    """the rules a search rarely meets, on hand-built logits: the lower flat index first among equal keys, a finished row's
    END at cost 0 and its other tokens at -FLT_MAX, only beam 0 at t = 0, len_out by parent, and logp the raw total while
    scores carry the penalised key"""
    lg = torch.log(torch.tensor([[0.4, 0.3, 0.3], [0.5, 0.25, 0.25], [0.6, 0.2, 0.2]], dtype=torch.float64))
    logp = torch.tensor([-1.0, -1.0, -2.0], dtype=torch.float64)
    fin = torch.tensor([False, False, True])
    o = dr.beam_step(lg, logp, fin, 0, 3, 0)
    assert o["parents"].tolist() == [[0, 0, 0]] and o["ids"].tolist() == [[0, 1, 2]]      # t = 0: row 0 only, ties by index
    o = dr.beam_step(lg, logp, fin, 1, 3, 0)
    # totals: row 0 (-1 + log .4, -1 + log .3, ...), row 1 (-1 + log .5, ...), row 2 finished: END -2, others -FLT_MAX
    # ranked: row 1's END (-1.69), row 0's END (-1.92), row 2's END (-2), row 0's token 1 (-2.20)
    assert o["parents"].tolist() == [[1, 0, 2]] and o["ids"].tolist() == [[0, 0, 0]]
    assert o["fin"].tolist() == [[True, True, True]]
    assert o["key"][0, 2 * 3 + 1].item() == -dr.FLT_MAX and o["key"][0, 2 * 3].item() == -2.0
    LP = bpo.length_penalty_table(1.0, 10, torch.float64)
    o = dr.beam_step(lg, logp, fin, 1, 3, 0, len_pen=LP, len_in=torch.tensor([2, 3, 4]))
    par, ids = o["parent_rows"].tolist(), o["ids"][0].tolist()
    assert o["len_out"].tolist() == [2 + par[k] + (0 if ids[k] == 0 or par[k] == 2 else 1) for k in range(3)]
    k0 = int(o["parents"][0, 0]) * 3 + int(o["ids"][0, 0])
    assert o["logp"][0].item() == o["total"][0, k0].item() != o["scores"][0].item()


def test_div_philox_uniforms_follow_the_stream_layout():
    """u of (row b, step t, token v) is word v & 3 of the counter (v >> 2, t, b, call): the dropout stream's layout (the
    host mirror of the dropout multipliers takes the same words)"""
    from latex_ocr_b200 import philox
    seed, call, B, V = 0x1234567890ABC, 3, 5, 13
    u = dr.div_philox_uniforms(seed, call, 2, B, V)
    m = philox.dropout_multipliers(seed, call, B, 3, V, 0.5)[:, 2]
    assert torch.equal(torch.from_numpy(m) > 0, u.float() >= 0.5)
    assert float(u.min()) >= 0 and float(u.max()) < 1


# ---------------------------------------------------------------------------------------------------------------------------------
# sampling
# ---------------------------------------------------------------------------------------------------------------------------------
_SAMPLE = [(1.0, 0, 1.0), (0.5, 0, 1.0), (2.0, 0, 1.0), (1.0, 1, 1.0), (1.0, V, 1.0), (1.0, 5, 0.6), (1.0, 0, 1e-6)]


@pytest.mark.parametrize("flavour", ["torch", "tf", "two_layer"])
@pytest.mark.parametrize("tau,top_k,top_p", _SAMPLE, ids=["t%g-k%d-p%g" % s for s in _SAMPLE])
def test_sampling_is_the_oracle(flavour, tau, top_k, top_p):
    n, N, R = 8, 2, 12
    encs = _encs([R] * N, 10)
    enc = torch.stack(encs)
    u = torch.rand(MAX_ITER + 2, N * n, V, generator=torch.Generator().manual_seed(11), dtype=torch.float64).clamp_min(1e-12)
    if flavour == "tf":
        p = _tf_params(12)
        cell, _, B = tf_flavour(p, encs, n)
        ocell, _ = so.tf_cell(p, enc, n)
    elif flavour == "torch":
        p = _torch_params(12)
        cell, _, B = torch_flavour(p, encs, n)
        ocell, _ = so.torch_cell(p, enc, n, START)
    else:
        p, p2 = _torch_params(12), _layer2_params(13)
        cell, _, B = torch_flavour(p, encs, n, p2)
        ocell, _ = so.decoder2_cell(p, p2, enc, n, START)
    ids, logp = sample_loop(cell, B, tau, top_k, top_p, u)
    w_ids, w_lp, _ = so.search(ocell, B, END, MAX_ITER, tau, top_k, top_p, u)
    assert torch.equal(ids, w_ids)
    _close(logp, w_lp)
    if top_k == 1 or top_p < 1e-3:                     # one token kept: the rows of an image draw alike at step 0
        assert all(len(set(ids[i * n:(i + 1) * n, 0].tolist())) == 1 for i in range(N))


def test_sampling_finished_rows_emit_end_and_add_nothing():
    x = torch.randn(3, V, dtype=torch.float64)
    u = torch.rand(3, V, dtype=torch.float64)
    logp = torch.tensor([-1.0, -2.0, -3.0], dtype=torch.float64)
    tok, lp, fin, _ = dr.sample(x, torch.tensor([True, False, True]), logp, 1.0, 0, 1.0, u, END)
    assert tok[0] == END and tok[2] == END and lp[0] == -1.0 and lp[2] == -3.0
    assert abs(lp[1] - (-2.0 + torch.log_softmax(x[1], -1)[tok[1]])) < 1e-12 and fin[0] and fin[2]


def test_sampling_uniforms_are_the_gumbel_stream():
    from latex_ocr_b200 import philox
    u = dr.philox_uniforms(77, 2, 3, 4, 10)
    assert torch.equal(u, torch.from_numpy(philox.gumbel_uniforms(77, 2, 4, 4, 10)[:, 3]))
