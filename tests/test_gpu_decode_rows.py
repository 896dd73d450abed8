"""-m gpu: decoding above 1,024 rows, and the split-count boundaries of the dense attention forward.

Decoding has no row cap: predict_batch of 256 images at beam 5 runs 1,280 rows.  Every attention launch keeps one ticket counter
per row in front of its split partials (include/latex_ocr_b200.h, lo_attention_workspace_bytes), so these tests decode batches
in which copies of the same images sit below and above row 1,024, and check every row against the CPU oracle
(oracle/ref_decode.py) run once per distinct image: tokens exactly, and the attention weights of every step against a float64
teacher-forced pass on those tokens.  The last test pins lo_attention_forward against float64 at the batch sizes where the split
count of each forward kernel changes."""
import pytest
import torch

from util import build_model, relerr

pytestmark = pytest.mark.gpu

V = 30
START = V - 2
POOL = 13                  # distinct images; row r holds image r % POOL, so rows 0 and 1024 hold different images (1024 % 13 = 10)
GREEDY_END, GREEDY_LEN = 7, 12
BEAM, BEAM_END, BEAM_LEN = 5, 5, 8


def _params(seed):
    """oracle parameters with a non-degenerate argmax: larger output layer and embedding (as in test_gpu_decode._setup)"""
    from oracle import ref_model as rm
    pe, pd = rm.init_params(V, seed=seed)
    g = torch.Generator().manual_seed(seed)
    pd["fc.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 0.5
    pd["embedding.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 1.0
    return pe, pd


def _rows(pool, N):
    """N images, copies of the pool in rotating order, and which pool image each one is"""
    idx = torch.arange(N) % pool.shape[0]
    return pool[idx].contiguous(), idx


class _Setup:
    def __init__(self, seed=21, H=32, W=64):
        from oracle import ref_decode as rd
        from oracle import ref_model as rm
        self.pe, self.pd = _params(seed)
        self.pool, _ = rm.synthetic_batch(POOL, H, W, V, 3, 5, seed=seed + 1)            # [13, 1, 32, 64]: R = 2 * 6 = 12
        self.enc = rm.encoder_forward(self.pe, self.pool).reshape(POOL, -1, 512)
        self.ids = rd.greedy_decode(self.pd, self.enc, START, GREEDY_END, GREEDY_LEN + 1)     # [13, steps]
        assert len({tuple(r.tolist()) for r in self.ids}) > 1        # rows of different images decode differently
        self._beam = {}
        self._al64 = None

    def alphas64(self):
        """float64 teacher-forced attention weights [13, steps, R] on the oracle's greedy tokens"""
        if self._al64 is None:
            from oracle import ref_model as rm
            p64 = {k: v.double() for k, v in self.pe.items()}
            d64 = {k: v.double() for k, v in self.pd.items()}
            enc = rm.encoder_forward(p64, self.pool.double()).reshape(POOL, -1, 512)
            n = self.ids.shape[1]
            caps = torch.cat([torch.full((POOL, 1), START, dtype=torch.long), self.ids], dim=1)
            lens = torch.full((POOL, 1), n + 1, dtype=torch.long)
            _, _, _, al, sort_ind = rm.decoder_forward(d64, enc, caps, lens)          # rows in sorted order
            self._al64 = torch.empty_like(al)
            self._al64[sort_ind] = al
        return self._al64

    def beam(self, fin):
        """oracle beam search per distinct image: ids [13, beam, steps], logp [13, beam]"""
        if fin not in self._beam:
            from oracle import ref_decode as rd
            want, wlp = rd.beam_decode(self.pd, self.enc, START, BEAM_END, beam=BEAM, max_iter=BEAM_LEN + 1, finalize=fin)
            self._beam[fin] = (want.permute(0, 2, 1).contiguous(), wlp)
        return self._beam[fin]


@pytest.fixture(scope="module")
def setup():
    return _Setup()


@pytest.fixture(scope="module")
def fp32_model(setup):
    return build_model(V, setup.pe, setup.pd, "fp32")


@pytest.fixture(scope="module")
def bf16_model(setup):
    return build_model(V, setup.pe, setup.pd, "bf16", impl="tc")


def _bad_rows(ok):
    bad = (~ok).nonzero().flatten()
    return "%d bad rows, first %s" % (bad.numel(), bad[:8].tolist())


def _check_greedy(setup, ids, al, idx):
    ok = (ids == setup.ids[idx]).all(dim=1)
    assert ok.all(), _bad_rows(ok)
    err = (al.double() - setup.alphas64()[idx]).abs().amax(dim=(1, 2))
    assert (err < 1e-5).all(), "%s, largest error %.3e" % (_bad_rows(err < 1e-5), err.max().item())


@pytest.mark.parametrize("N,pipe", [(1024, 1), (1025, 1), (1300, 1), (1300, 0)])
def test_dense_greedy_every_row_matches_the_oracle(setup, fp32_model, N, pipe):
    from latex_ocr_b200 import _lib, decode
    img, idx = _rows(setup.pool, N)
    with _lib.option(att_pipe=pipe):
        ids, al = decode.greedy_decode(fp32_model, img, START, GREEDY_END, GREEDY_LEN, return_attention=True)
    assert ids.shape == (N, setup.ids.shape[1]) and al.shape == (N, setup.ids.shape[1], 12)
    _check_greedy(setup, ids, al, idx)


@pytest.mark.parametrize("n_img", [205, 256])
def test_dense_beam_every_row_matches_the_oracle(setup, fp32_model, n_img):
    """205 and 256 images at beam 5: 1,025 and 1,280 rows"""
    from latex_ocr_b200 import decode
    img, idx = _rows(setup.pool, n_img)
    for fin in ("reference", "backtrack"):
        want, wlp = setup.beam(fin)
        got, glp = decode.beam_decode(fp32_model, img, START, BEAM_END, beam_size=BEAM, max_length_formula=BEAM_LEN, finalize=fin)
        assert got.shape == (n_img,) + tuple(want.shape[1:]), fin
        ok = (got == want[idx]).flatten(1).all(dim=1)
        assert ok.all(), (fin, _bad_rows(ok))
        assert (glp - wlp[idx]).abs().max().item() < 1e-3 * max(1.0, wlp.abs().max().item()), fin


def _tensor_and_list_agree(m, img, beam):
    from latex_ocr_b200 import decode
    if beam == 1:
        ids_t, al_t = decode.greedy_decode(m, img, START, GREEDY_END, GREEDY_LEN, return_attention=True)
        ids_l, al_l = decode.greedy_decode(m, list(img), START, GREEDY_END, GREEDY_LEN, return_attention=True)
        assert torch.equal(ids_t, ids_l)
        assert torch.equal(al_t, torch.stack(al_l))
        return ids_t
    ids_t, lp_t = decode.beam_decode(m, img, START, BEAM_END, BEAM, BEAM_LEN)
    ids_l, lp_l = decode.beam_decode(m, list(img), START, BEAM_END, BEAM, BEAM_LEN)
    assert torch.equal(ids_t, ids_l)
    assert torch.equal(lp_t, lp_l)
    return ids_t


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("n_img,beam", [(1300, 1), (256, BEAM)])
def test_tensor_path_equals_list_path_bit_for_bit_above_1024_rows(setup, fp32_model, bf16_model, precision, n_img, beam):
    """The list path (per-image region counts) gives every row the partition of the dense launch: same bits."""
    m = fp32_model if precision == "fp32" else bf16_model
    img, idx = _rows(setup.pool, n_img)
    ids = _tensor_and_list_agree(m, img, beam)
    if precision == "fp32" and beam == 1:
        assert torch.equal(ids, setup.ids[idx])


def test_tensor_path_equals_list_path_at_cfg2_size_above_1024_rows(setup, bf16_model):
    """cfg #2 images (128 x 512 px, R = 868), 205 of them at beam 5: 1,025 rows"""
    from oracle import ref_model as rm
    pool, _ = rm.synthetic_batch(POOL, 128, 512, V, 3, 5, seed=90)
    img, _ = _rows(pool, 205)
    assert bf16_model.encoder.out_hw(128, 512) == (14, 62)
    _tensor_and_list_agree(bf16_model, img, BEAM)


def test_tensor_path_equals_list_path_with_three_splits_through_the_ticket_combine(setup, fp32_model):
    """att_nsplit=3 without clusters: every row's three splits meet at its ticket counter, rows 1024.. included"""
    from latex_ocr_b200 import _lib
    img, idx = _rows(setup.pool, 1300)
    with _lib.option(att_nsplit=3, att_cluster=0):
        ids = _tensor_and_list_agree(fp32_model, img, 1)
    assert torch.equal(ids, setup.ids[idx])


def test_back_to_back_calls_on_one_model_repeat_their_bits(setup):
    """Dense decode workspaces of different row counts on one model, then list decodes that reuse one ragged workspace"""
    from latex_ocr_b200 import decode
    m = build_model(V, setup.pe, setup.pd, "fp32")
    first = {}
    for N in (600, 1300, 600, 1300):
        img, idx = _rows(setup.pool, N)
        ids, al = decode.greedy_decode(m, img, START, GREEDY_END, GREEDY_LEN, return_attention=True)
        _check_greedy(setup, ids, al, idx)
        if N in first:
            assert torch.equal(ids, first[N][0]) and torch.equal(al, first[N][1]), N
        else:
            first[N] = (ids, al)
    n_ws = None
    for N in (1300, 500, 1300):
        img, idx = _rows(setup.pool, N)
        ids, al = decode.greedy_decode(m, list(img), START, GREEDY_END, GREEDY_LEN, return_attention=True)
        al = torch.stack(al)
        _check_greedy(setup, ids, al, idx)
        if N in first:         # the list path reproduces the dense path's bits
            assert torch.equal(ids, first[N][0]) and torch.equal(al, first[N][1]), N
        n_ws = len(m.decoder._ws) if n_ws is None else n_ws
        assert len(m.decoder._ws) == n_ws               # the ragged workspace of the first call is reused


# ---- split-count boundaries of lo_attention_forward: att_pipe_splits = 264 // B (capped at 8 with clusters),
#      att_splits = ceil(444 / B)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("pipe,cluster", [(0, 1), (1, 1), (1, 2)])
@pytest.mark.parametrize("R", [1, 2, 17, 101])
@pytest.mark.parametrize("B", [1, 2, 33, 34, 132, 133, 443, 444, 512])
def test_attention_forward_at_split_boundaries(B, R, pipe, cluster, dtype):
    from latex_ocr_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(1000 * B + R)
    C = A = 512
    enc = torch.randn(B, R, C, device="cuda", generator=g).to(dtype)
    att1 = torch.randn(B, R, A, device="cuda", generator=g).to(dtype)
    att2 = torch.randn(B, A + 16, device="cuda", generator=g)[:, :A]          # strided rows
    wf = torch.randn(A, device="cuda", generator=g) * 0.2
    gate_pre = torch.randn(B, C, device="cuda", generator=g)
    gp0 = gate_pre.clone()
    alpha = torch.zeros(B, R, device="cuda")
    ctx = torch.zeros(B, C, device="cuda")
    gctx = torch.zeros(B, C, device="cuda")
    work = torch.zeros(int(L.lo_attention_workspace_bytes(B, C)), dtype=torch.uint8, device="cuda")
    with _lib.option(att_pipe=pipe, att_cluster=cluster):
        for _ in range(2):     # second launch checks that the ticket counters were reset
            gate_pre.copy_(gp0)
            _lib.check(L.lo_attention_forward(_lib.ptr(att1), _lib.ptr(enc), _lib.dt_of(enc), _lib.ptr(att2), att2.stride(0),
                                              _lib.ptr(wf), _lib.ptr(alpha), R, _lib.ptr(ctx), _lib.ptr(gate_pre), C, _lib.ptr(gctx),
                                              B, R, A, C, _lib.ptr(work), _lib.stream_ptr()))
            torch.cuda.synchronize()
    assert not work[:4 * B].any()                    # every row's counter is back at zero
    e = (torch.relu(att1.double() + att2.double()[:, None, :]) * wf.double()).sum(-1)
    al = torch.softmax(e, dim=1)
    cx = torch.einsum("br,brc->bc", al, enc.double())
    if R == 1:
        # one region: the splits without a region hold M = -inf and must drop out of the combine entirely
        assert torch.equal(alpha, torch.ones_like(alpha))
        assert relerr(ctx, enc[:, 0].float()) < 1e-6
    assert relerr(alpha, al.float()) < 2e-5
    assert relerr(ctx, cx.float()) < 2e-5
    assert relerr(gate_pre, torch.sigmoid(gp0)) < 1e-6
    assert relerr(gctx, (torch.sigmoid(gp0.double()) * cx).float()) < 2e-5
