"""Float64 restatement of one decode step of the library's decode loops (greedy_loop, sample_loop and beam_loop in
csrc/lo_decoder.cu), split the way the kernels split it, so that a test can feed each piece the operands one kernel read.

The step before the choice is the flavour's own (tests/decoder_step_ref.py, tests/tfdec_step_ref.py; the two-layer decoder adds
tests/lstmseq_step_ref.py's layer); what decode adds is the row-to-image map: row b reads image b // rows_per_img, over that image's
own region count (reg_off), and starts from the mean of that image's own regions (``region_means``, ``rows_of``).

The choices, on given fp32 logits [B][V] (as float64) and state:
  * greedy (argmax_kernel): the lowest-index argmax; finished |= token == END; a finished row keeps emitting its argmax (the
    reference's greedy cell decodes on after END; the caller truncates).
  * sampling (sample_step_kernel): tests/sample_oracle.py's keep_mask / draw; logp += log_softmax(x)[token] at temperature 1;
    a finished row emits END and adds nothing.
  * beam search (beam_step_kernel, one image of ``beam`` rows): lp = log_softmax(logits) per row; a finished row's lp is
    [END: 0, else: -FLT_MAX]; total = logp + lp (+ the diversity penalty log(gamma) * rank inside the row where prob > u, ranks
    with the lower index first among equals); only beam 0 at t = 0; key = total / len_pen[len_in + (finished or END ? 0 : 1)]
    + cov_term, a finished row's non-END keys -FLT_MAX; top-k by repeated extraction, the lower flat index first among equal
    keys; id = idx % V, parent = idx // V; logp = the winner's total, scores = its key, len_out = len_in[parent] + (finished
    parent or END ? 0 : 1).
  * coverage (beam_coverage_kernel): cov_out[b] = cov_in[parent_rows[b]] (0 at t = 0) + alpha_t[b] where row b is unfinished,
    over the image's own regions; term[b] = beta * sum_r ln(min(max(cov_r, 1e-30), 1)).

Every function returns float64 (ids int64) and, where a sum is formed, S: the sum of the magnitudes of its terms.
"""
import math

import numpy as np
import torch

import sample_oracle as so

FLT_MAX = 3.4028234663852886e38


# ---------------------------------------------------------------------------------------------------------------------------------
# the row-to-image map
# ---------------------------------------------------------------------------------------------------------------------------------
def rows_of(x, rows_per_img):
    """per-image values [N][...] -> per-row values [N * rows_per_img][...] (row b reads image b // rows_per_img)"""
    return x.repeat_interleave(rows_per_img, dim=0)


def region_means(enc, counts):
    """(mean [N][C], S [N][C]) of the packed encoder rows enc [regions][C] of images of ``counts`` regions each: every image's
    mean over its own regions only"""
    out, S, o = [], [], 0
    for n in counts:
        e = enc[o:o + n]
        out.append(e.sum(0) / n)
        S.append(e.abs().sum(0) / n)
        o += n
    return torch.stack(out), torch.stack(S)


# ---------------------------------------------------------------------------------------------------------------------------------
# greedy
# ---------------------------------------------------------------------------------------------------------------------------------
def greedy(logits, finished, end_id):
    """(tokens [B], finished [B] bool): the lowest-index argmax of every row; finished |= token == END"""
    tok = torch.argmax(logits, dim=-1)                  # the first maximum
    return tok, finished | (tok == end_id)


# ---------------------------------------------------------------------------------------------------------------------------------
# sampling
# ---------------------------------------------------------------------------------------------------------------------------------
def sample(logits, finished, logp, tau, top_k, top_p, u, end_id):
    """(tokens [B], logp [B], finished [B] bool, margin): one step of sampling decode; u [B][V] the uniforms of the step.
    margin: the least top-p margin of the unfinished rows (sample_oracle.keep_mask)."""
    x = logits.double().cpu().numpy()
    uu = torch.as_tensor(u).double().cpu().numpy()
    B = x.shape[0]
    tok = np.full(B, end_id, dtype=np.int64)
    lp = logp.double().cpu().numpy().copy()
    fin = finished.cpu().numpy().astype(bool)
    margin = math.inf
    for b in range(B):
        if fin[b]:
            continue
        kept, m = so.keep_mask(x[b], tau, top_k, top_p)
        margin = min(margin, m)
        tok[b] = so.draw(x[b], tau, kept, uu[b])
        z = x[b] - x[b].max()
        lp[b] += z[tok[b]] - math.log(np.exp(z).sum())
    dev = logits.device
    tok = torch.from_numpy(tok).to(dev)
    return tok, torch.from_numpy(lp).to(dev), finished | (tok == end_id), margin


def philox_uniforms(seed, call, t, B, V):
    """[B][V] float64: the uniforms u of sampling decode's Gumbel draws at step t under the Philox state {seed, call}, exactly
    as sample_step_kernel takes them (latex_ocr_b200/philox.py gumbel_uniforms)"""
    from latex_ocr_b200 import philox
    return torch.from_numpy(philox.gumbel_uniforms(seed, call, B, t + 1, V)[:, t])


# ---------------------------------------------------------------------------------------------------------------------------------
# beam search
# ---------------------------------------------------------------------------------------------------------------------------------
def div_philox_uniforms(seed, call, t, B, V):
    """[B][V] float64: the diversity uniforms of beam step t, row b, token v under the Philox state {seed, call}: word v & 3 of
    philox4x32_10(counter (v >> 2, t, b, call), key (seed lo, seed hi)), u = (word >> 8) 2^-24 (the dropout stream's layout)"""
    from latex_ocr_b200 import philox
    b = np.arange(B, dtype=np.uint64)[:, None]
    v4 = np.arange((V + 3) // 4, dtype=np.uint64)[None, :]
    w = philox.philox4x32_10(v4 + 0 * b, np.uint64(t) + 0 * b + 0 * v4, b + 0 * v4, np.uint64(call), seed & 0xFFFFFFFF,
                             (seed >> 32) & 0xFFFFFFFF)
    x = np.stack(w, axis=-1).reshape(B, -1)[:, :V]
    return torch.from_numpy((x >> np.uint64(8)).astype(np.float64) * 2.0 ** -24)


def log_softmax(logits):
    """(lp [B][V], lse [B])"""
    lse = torch.logsumexp(logits, dim=-1)
    return logits - lse[:, None], lse


def div_ranks(total):
    """rank of every candidate inside its row [..][V] (0 = the largest; the lower index first among equals)"""
    order = torch.argsort(total, dim=-1, descending=True, stable=True)
    return torch.argsort(order, dim=-1).double()


def beam_step(logits, logp, finished, t, beam, end_id, log_gamma=0.0, div_prob=0.0, div_u=None, len_pen=None, cov_term=None,
              len_in=None):
    """One beam_step_kernel launch over B = n_img * beam rows.  logits [B][V], logp [B], finished [B] bool (after step t-1),
    div_u [B][V] (with div_prob > 0 and log_gamma != 0), len_pen the fp32 table as float64, cov_term [B] the coverage terms,
    len_in [B] (the lengths after step t-1; read when penalties are on).  Returns a dict: ids, parents [n_img][beam], fin,
    next_tok, parent_rows, logp, scores, len_out [B]; and per candidate (flat index k * V + v of the image) total, key, lp, lse
    [n_img][beam * V], the ranks [n_img][beam * V] (0 without diversity) and nb (1 at t = 0)."""
    B, V = logits.shape
    N = B // beam
    dev = logits.device
    lp, lse = log_softmax(logits.double())
    fin = finished.bool().to(dev)
    is_end = torch.arange(V, device=dev) == end_id
    lp = torch.where(fin[:, None], torch.where(is_end, 0.0, -FLT_MAX).double().expand(B, V), lp)
    total = logp.double()[:, None] + lp
    masked = fin[:, None] & ~is_end[None, :]
    total = torch.where(masked, torch.full_like(total, -FLT_MAX), total)          # -FLT_MAX + logp rounds to -FLT_MAX in fp32
    rank = torch.zeros_like(total)
    if div_prob > 0 and log_gamma != 0:
        nb = 1 if t == 0 else beam
        tv = total.view(N, beam, V)
        rank = div_ranks(tv).view(B, V)
        total = total + torch.where(div_prob > div_u.double().to(dev), log_gamma * rank, torch.zeros_like(rank))
    pen = len_in is not None
    if pen:
        lin = torch.zeros(B, dtype=torch.long, device=dev) if t == 0 else len_in.long().to(dev)
        new_len = lin[:, None] + (~fin[:, None] & ~is_end[None, :]).long()
        key = total
        if len_pen is not None:
            key = key / len_pen.double().to(dev)[new_len]
        if cov_term is not None:
            key = key + cov_term.double().to(dev)[:, None]
        key = torch.where(masked, torch.full_like(key, -FLT_MAX), key)
    else:
        key = total
    nb = 1 if t == 0 else beam
    key3 = key.view(N, beam, V)[:, :nb].reshape(N, nb * V)
    tot3 = total.view(N, beam, V)[:, :nb].reshape(N, nb * V)
    ids, parents, vals, carried = [], [], [], []
    kk = key3.clone()
    ar = torch.arange(N, device=dev)
    for _ in range(beam):
        m = kk.max(dim=1).values
        i = (kk == m[:, None]).double().argmax(dim=1)             # the first maximum: the lower flat index
        ids.append(i % V)
        parents.append(i // V)
        vals.append(m)
        carried.append(tot3[ar, i])
        kk[ar, i] = -math.inf
    ids, parents = torch.stack(ids, 1), torch.stack(parents, 1)
    rows = parents + ar[:, None] * beam
    fin_par = fin[rows.reshape(-1)].view(N, beam)
    fin_new = fin_par | (ids == end_id)
    out = dict(ids=ids, parents=parents, fin=fin_new, next_tok=ids.reshape(-1), parent_rows=rows.reshape(-1),
               logp=torch.stack(carried, 1).reshape(-1), scores=torch.stack(vals, 1).reshape(-1),
               total=tot3, key=key3, lp=lp.view(N, beam, V)[:, :nb].reshape(N, nb * V),
               lse=lse.view(N, beam)[:, :nb].repeat_interleave(V, dim=1), rank=rank.view(N, beam, V)[:, :nb].reshape(N, nb * V),
               nb=nb)
    if pen:
        out["len_out"] = (lin[rows.reshape(-1)].view(N, beam) + (~fin_par & (ids != end_id)).long()).reshape(-1)
    return out


def coverage(alpha_t, cov_in, parent_rows, finished, counts, beam, t, beta):
    """(cov_out [B][R], term [B], S_term [B]): beam_coverage_kernel.  alpha_t [B][R] the attention rows of step t, cov_in [B][R]
    step t-1's coverage (ignored at t = 0), parent_rows [B] step t-1's selection, finished [B] after step t-1, counts: every
    image's own region count.  Entries at or past an image's count are not written (cov_out holds NaN there)."""
    B, R = alpha_t.shape
    dev = alpha_t.device
    cov = torch.full((B, R), math.nan, dtype=torch.float64, device=dev)
    term = torch.zeros(B, dtype=torch.float64, device=dev)
    S = torch.zeros_like(term)
    for b in range(B):
        n = counts[b // beam]
        c = torch.zeros(n, dtype=torch.float64, device=dev) if t == 0 else cov_in[int(parent_rows[b]), :n].double()
        if not bool(finished[b]):
            c = c + alpha_t[b, :n].double()
        cov[b, :n] = c
        lg = torch.log(c.clamp(1e-30, 1.0))
        term[b] = beta * lg.sum()
        S[b] = beta * lg.abs().sum()
    return cov, term, S
