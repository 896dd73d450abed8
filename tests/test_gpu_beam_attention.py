"""-m gpu: the attention weights of beam-search hypotheses in both decoder flavours (lo_beam_backtrack).

The kernel alone is a copy: its ids and attention rows equal a torch gather along the parents bit for bit.  Through the decoders,
under finalize='reference' every slot's rows equal the CPU oracle's per-slot rows, and under 'backtrack' every hypothesis's rows
equal a float64 teacher-forced pass over its own tokens (oracle/ref_decode.py, oracle/ref_tf_model.py)."""
import ctypes

import pytest
import torch

import beam_oracle as bo
from util import Cfg, build_model

pytestmark = pytest.mark.gpu

V = 30
START, END = V - 2, 5
BEAM, LEN = 5, 8
POOL = 13                   # distinct images of the row-count tests; row r holds image r % POOL


# ------------------------------------------------------------------------------------------------ the kernel alone
def _kernel_case(n_img, beam, n, R, counts, mode, seed):
    from latex_ocr_b200 import _lib, decode
    from oracle import ref_decode as rd
    g = torch.Generator().manual_seed(seed)
    steps = n + 3                                    # ids / parents are [n_img][steps][beam]: n of them are read
    ids = torch.randint(0, 1000, (n_img, steps, beam), generator=g)
    parents = torch.randint(0, beam, (n_img, steps, beam), generator=g)
    alphas = torch.rand(n_img * beam, steps, R, generator=g)
    a = None
    if counts is not None:                           # the decode args' region offsets, as set_region_offsets leaves them
        a = _lib.DecoderArgs()
        off = decode.region_offsets(counts)
        host, dev = (ctypes.c_int32 * len(off))(), torch.zeros(len(off), dtype=torch.int32, device="cuda")
        decode.set_region_offsets(a, host, dev, off)
    l0 = _lib.launch_count()
    got_ids, got_att = decode.beam_hypotheses(ids.cuda()[:, :n], parents.cuda()[:, :n], mode, a, alphas.cuda())
    assert _lib.launch_count() - l0 == 1
    want_ids = (ids[:, :n] if mode == "reference" else rd.backtrack(ids[:, :n], parents[:, :n])).permute(0, 2, 1)
    want_att = bo.hypothesis_attention(alphas[:, :n], parents[:, :n], mode)
    if counts is not None:
        for i, c in enumerate(counts):
            want_att[i, :, :, c:] = 0
    assert torch.equal(got_ids.cpu(), want_ids)
    assert torch.equal(got_att.cpu(), want_att)
    return got_att


@pytest.mark.parametrize("beam", [1, 2, 5, 16])
@pytest.mark.parametrize("n", [1, 152])
@pytest.mark.parametrize("R", [12, 13])
@pytest.mark.parametrize("mode", ["reference", "backtrack"])
def test_kernel_equals_a_torch_gather(beam, n, R, mode):
    _kernel_case(7, beam, n, R, None, mode, seed=beam * 1000 + n + R)
    counts = [1, R, 3, R - 1, 2, R, 5]               # ragged, with a count of 1 and counts inside a 16-byte group
    att = _kernel_case(7, beam, n, R, counts, mode, seed=beam * 1000 + n + R + 1)
    assert (att[0, :, :, 1:] == 0).all()


# ------------------------------------------------------------------------------------------------ torch flavour
def _params(seed):
    """oracle parameters with a non-degenerate argmax (as in test_gpu_ragged_decode)"""
    from oracle import ref_model as rm
    pe, pd = rm.init_params(V, seed=seed)
    g = torch.Generator().manual_seed(seed)
    pd["fc.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 0.5
    pd["embedding.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 1.0
    return pe, pd


def _mixed(seed, shapes=((32, 64), (48, 96), (32, 200), (48, 64), (32, 128)), per=2):
    from oracle import ref_model as rm
    groups = [rm.synthetic_batch(per, H, W, V, 3, 5, seed=seed + k)[0] for k, (H, W) in enumerate(shapes)]
    return [groups[k][i] for i in range(per) for k in range(len(shapes))]


def _enc(pe, img):
    """oracle encoder output [N, R, 512] of a batch [N,1,H,W]"""
    from oracle import ref_model as rm
    return rm.encoder_forward(pe, img).reshape(img.shape[0], -1, 512)


def _tf64(pe, pd, img, hyps):
    """float64 teacher-forced attention [N, beam, n, R] over hypotheses [N, beam, n] of the batch img"""
    p64 = {k: v.double() for k, v in pd.items()}
    return bo.teacher_forced_attention(p64, _enc({k: v.double() for k, v in pe.items()}, img.double()), START, hyps)


@pytest.fixture(scope="module")
def torch_setup():
    pe, pd = _params(21)
    return pe, pd, build_model(V, pe, pd, "fp32")


def test_torch_reference_attention_equals_the_oracle_slot_rows(torch_setup):
    from latex_ocr_b200 import decode
    from oracle import ref_decode as rd
    from oracle import ref_model as rm
    pe, pd, m = torch_setup
    img, _ = rm.synthetic_batch(6, 32, 64, V, 3, 5, seed=3)
    ids, lp, att = decode.beam_decode(m, img, START, END, BEAM, LEN, return_attention=True)
    want, _, alphas, parents = bo.recorded_beam("torch", pd, _enc(pe, img), V, START, END, BEAM, LEN + 1)
    assert torch.equal(ids, want.permute(0, 2, 1))
    assert att.shape == ids.shape + (12,) and att.device.type == "cpu"
    assert (att - bo.hypothesis_attention(alphas, parents, "reference")).abs().max().item() < 1e-5
    assert (att.sum(dim=3) - 1).abs().max().item() < 1e-5
    # attention off: the same ids and log-probs, bit for bit
    ids0, lp0 = decode.beam_decode(m, img, START, END, BEAM, LEN)
    assert torch.equal(ids, ids0) and torch.equal(lp, lp0)


@pytest.mark.parametrize("n_img", [6, 205, 256])
def test_torch_backtrack_attention_is_the_teacher_forced_attention(torch_setup, n_img):
    """205 and 256 images at beam 5: 1,025 and 1,280 rows, copies of 13 distinct images"""
    from latex_ocr_b200 import _lib, decode
    from oracle import ref_model as rm
    pe, pd, m = torch_setup
    pool, _ = rm.synthetic_batch(POOL, 32, 64, V, 3, 5, seed=22)
    idx = torch.arange(n_img) % POOL
    img = pool[idx].contiguous()
    ids0, lp0 = decode.beam_decode(m, img, START, END, BEAM, LEN, finalize="backtrack")
    l0 = _lib.launch_count()
    ids, lp, att = decode.beam_decode(m, img, START, END, BEAM, LEN, finalize="backtrack", return_attention=True)
    l1 = _lib.launch_count()
    decode.beam_decode(m, img, START, END, BEAM, LEN, finalize="backtrack")
    assert l1 - l0 == _lib.launch_count() - l1          # attention adds no launch: the ids come from the same kernel
    assert torch.equal(ids, ids0) and torch.equal(lp, lp0)
    k = min(n_img, POOL)
    assert torch.equal(ids, ids[:k][idx % k])             # every copy of an image decodes alike
    want = _tf64(pe, pd, pool[:k], ids[:k])
    err = (att.double() - want[idx % k]).abs().amax(dim=(1, 2, 3))
    assert (err < 1e-5).all(), err.max().item()
    assert (att.sum(dim=3) - 1).abs().max().item() < 1e-5


@pytest.mark.parametrize("fin", ["reference", "backtrack"])
def test_torch_list_path(torch_setup, fin):
    from latex_ocr_b200 import _lib, decode
    from oracle import ref_model as rm
    pe, pd, m = torch_setup
    # one size: the list path equals the tensor path bit for bit
    img, _ = rm.synthetic_batch(8, 32, 64, V, 3, 5, seed=31)
    ids_t, lp_t, att_t = decode.beam_decode(m, img, START, END, BEAM, LEN, finalize=fin, return_attention=True)
    ids_l, lp_l, att_l = decode.beam_decode(m, list(img), START, END, BEAM, LEN, finalize=fin, return_attention=True)
    assert torch.equal(ids_t, ids_l) and torch.equal(lp_t, lp_l)
    assert torch.equal(att_t, torch.stack(att_l))
    # mixed sizes: every image's attention is its own, over its own regions, and what it gets decoded alone
    imgs = _mixed(40)
    with _lib.option(att_nsplit=3):                       # a fixed split partitions every row alike whatever the composition
        ids, lp, att = decode.beam_decode(m, imgs, START, END, BEAM, LEN, finalize=fin, return_attention=True)
        ids0, lp0 = decode.beam_decode(m, imgs, START, END, BEAM, LEN, finalize=fin)
        assert torch.equal(ids, ids0) and torch.equal(lp, lp0)
        assert len(att) == len(imgs)
        for i in (0, 3, 7):
            x = imgs[i]
            h, w = m.encoder.out_hw(x.shape[1], x.shape[2])
            assert att[i].shape == (BEAM, ids.shape[2], h * w)
            assert (att[i].sum(dim=2) - 1).abs().max().item() < 1e-5
            ids_a, _, att_a = decode.beam_decode(m, [x], START, END, BEAM, LEN, finalize=fin, return_attention=True)
            n = ids_a.shape[2]
            assert torch.equal(ids[i, :, :n], ids_a[0])
            assert torch.equal(att[i][:, :n], att_a[0])
            if fin == "backtrack":
                want = _tf64(pe, pd, x.unsqueeze(0), ids_a)[0]
                assert (att_a[0].double() - want).abs().max().item() < 1e-5


def test_torch_beam_1_equals_the_greedy_export(torch_setup):
    """beam 1 runs the same step kernels on the same state as greedy decode (the reorder gathers rows by the identity)"""
    from latex_ocr_b200 import decode
    from oracle import ref_model as rm
    _, _, m = torch_setup
    img, _ = rm.synthetic_batch(9, 32, 64, V, 3, 5, seed=41)
    ids_g, att_g = decode.greedy_decode(m, img, START, END, LEN, return_attention=True)
    for fin in ("reference", "backtrack"):
        ids_b, _, att_b = decode.beam_decode(m, img, START, END, 1, LEN, finalize=fin, return_attention=True)
        assert torch.equal(ids_b[:, 0], ids_g)
        assert torch.equal(att_b[:, 0], att_g)


def test_torch_bf16_ids_unchanged_and_attention_near_fp32(torch_setup):
    """bf16 storage (wgmma / mma.sync GEMMs): the attention call returns the attention-off call's ids exactly.  Its attention weights
    are compared with the fp32 model's on the hypotheses whose tokens both precisions agree on: within 3e-2 absolute, the bound
    smoke() uses for the bf16 loss — enc, att1 and h enter the scores as bf16 (8 significant bits), and a softmax weight moves by
    about its own size times the score error."""
    from latex_ocr_b200 import decode
    from oracle import ref_model as rm
    pe, pd, m32 = torch_setup
    m16 = build_model(V, pe, pd, "bf16", impl="tc")
    img, _ = rm.synthetic_batch(40, 32, 64, V, 3, 5, seed=51)
    for fin in ("reference", "backtrack"):
        ids0, lp0 = decode.beam_decode(m16, img, START, END, BEAM, LEN, finalize=fin)
        ids, lp, att = decode.beam_decode(m16, img, START, END, BEAM, LEN, finalize=fin, return_attention=True)
        assert torch.equal(ids, ids0) and torch.equal(lp, lp0)
        ids32, _, att32 = decode.beam_decode(m32, img, START, END, BEAM, LEN, finalize=fin, return_attention=True)
        if ids32.shape != ids.shape:
            continue
        same = (ids32 == ids).all(dim=2)
        assert same.float().mean().item() > 0.5
        assert (att[same] - att32[same]).abs().max().item() < 3e-2


# ------------------------------------------------------------------------------------------------ TensorFlow flavour
TF_V = 40
SHAPES = ((4, 8), (6, 12), (4, 25), (6, 8), (4, 16))


def _tf_params(seed):
    from oracle import ref_tf_model as tfm
    p = tfm.init_params_tf(TF_V, seed=seed)
    p["y_W_o"] = p["y_W_o"] * 4.0
    return p


def _tf_decoder(p, beam, **kw):
    from latex_ocr_b200.tf_decoder import Decoder
    cfg = Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=10,
              decoding="beam_search", beam_size=beam, **kw)
    dec = Decoder(cfg, TF_V, END, device="cuda", precision="fp32", impl="simt")
    dec.load_tf_variables(p)
    return dec


def _tf_mixed(seed, per=2):
    g = torch.Generator().manual_seed(seed)
    groups = [[torch.relu(torch.randn(h * w, 512, generator=g)) * 0.7 for _ in range(per)] for h, w in SHAPES]
    return [groups[k][i] for i in range(per) for k in range(len(SHAPES))]


@pytest.mark.parametrize("beam", [1, 2, 5])
@pytest.mark.parametrize("div", [False, True])
def test_tf_attention_against_the_oracle(beam, div):
    from oracle import ref_decode as rd
    from oracle import ref_tf_model as tfm
    p = _tf_params(7)
    p64 = {k: v.double() for k, v in p.items()}
    kw = {"div_gamma": 0.5, "div_prob": 0.7} if div else {}
    dec = _tf_decoder(p, beam, **kw)
    L = dec.max_length_formula
    g = torch.Generator().manual_seed(8)
    enc = torch.relu(torch.randn(6, 96, 512, generator=g)) * 0.7
    u = torch.rand(L + 2, 6 * beam, TF_V, generator=torch.Generator().manual_seed(77)) if div else None
    out0, lp0 = dec.decode(enc.cuda(), div_u=u, return_log_probs=True)
    want, _, alphas, parents = bo.recorded_beam("tf", p, enc, TF_V, END, beam, L + 1, div_u=u, **kw)
    # reference finalize: today's ids, each slot's own rows
    out, lp, att = dec.decode(enc.cuda(), div_u=u, return_log_probs=True, return_attention=True)
    assert torch.equal(out.ids, out0.ids) and torch.equal(lp, lp0)
    assert torch.equal(out.ids.cpu(), want)
    assert (att.cpu() - bo.hypothesis_attention(alphas, parents, "reference")).abs().max().item() < 1e-5
    # backtrack: lineage-consistent ids and the teacher-forced attention of each hypothesis
    out_b, att_b = dec.decode(enc.cuda(), div_u=u, return_attention=True, finalize="backtrack")
    assert torch.equal(out_b.ids.cpu(), rd.backtrack(want, parents))
    hyps = out_b.ids.cpu().permute(0, 2, 1)
    tf = bo.tf_teacher_forced_attention(p64, enc.double(), hyps)
    assert (att_b.cpu().double() - tf).abs().max().item() < 1e-5
    assert (att_b.sum(dim=3) - 1).abs().max().item() < 1e-5
    if beam == 1 and not div:
        from latex_ocr_b200.tf_decoder import Decoder
        gdec = Decoder(Cfg(attn_cell_config=dict(dec._config.attn_cell_config), max_length_formula=10, decoding="greedy"), TF_V, END,
                       device="cuda", precision="fp32", impl="simt")
        gdec.load_tf_variables(p)
        out_g, att_g = gdec.decode(enc.cuda(), return_attention=True)
        assert torch.equal(out_g.ids, out_b.ids[:, :, 0]) and torch.equal(att_g, att_b[:, 0])


@pytest.mark.parametrize("fin", ["reference", "backtrack"])
def test_tf_list_path(fin):
    from latex_ocr_b200 import _lib
    from oracle import ref_tf_model as tfm
    p = _tf_params(9)
    dec = _tf_decoder(p, BEAM)
    g = torch.Generator().manual_seed(10)
    enc = (torch.relu(torch.randn(8, 96, 512, generator=g)) * 0.7).cuda()
    out_t, att_t = dec.decode(enc, return_attention=True, finalize=fin)
    out_l, att_l = dec.decode(list(enc), return_attention=True, finalize=fin)
    assert torch.equal(out_t.ids, out_l.ids) and torch.equal(att_t, torch.stack(att_l))
    encs = _tf_mixed(20)
    with _lib.option(att_nsplit=3):
        out, lp, att = dec.decode([e.cuda() for e in encs], return_log_probs=True, return_attention=True, finalize=fin)
        out0, lp0 = dec.decode([e.cuda() for e in encs], return_log_probs=True, finalize=fin)
        assert torch.equal(out.ids, out0.ids) and torch.equal(lp, lp0)
        for i in (0, 2, 6):
            e = encs[i]
            assert att[i].shape == (BEAM, out.ids.shape[1], e.shape[0])
            assert (att[i].sum(dim=2) - 1).abs().max().item() < 1e-5
            out_a, att_a = dec.decode([e.cuda()], return_attention=True, finalize=fin)
            n = out_a.ids.shape[1]
            assert torch.equal(out.ids[i, :n], out_a.ids[0])
            assert torch.equal(att[i][:, :n], att_a[0])
            if fin == "backtrack":
                want = bo.tf_teacher_forced_attention({k: v.double() for k, v in p.items()}, e[None].double(),
                                                    out_a.ids.cpu().permute(0, 2, 1))[0]
                assert (att_a[0].cpu().double() - want).abs().max().item() < 1e-5


def test_tf_bf16_ids_unchanged():
    """bf16: the attention call returns the attention-off call's ids exactly; its weights sum to 1 per row to bf16 accuracy of the
    scores (fp32 softmax)."""
    from latex_ocr_b200.tf_decoder import Decoder
    p = _tf_params(11)
    cfg = Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=10,
              decoding="beam_search", beam_size=BEAM)
    dec = Decoder(cfg, TF_V, END, device="cuda", precision="bf16", impl="tc")
    dec.load_tf_variables(p)
    enc = (torch.relu(torch.randn(40, 96, 512, generator=torch.Generator().manual_seed(12))) * 0.7).cuda()
    for fin in ("reference", "backtrack"):
        out0, lp0 = dec.decode(enc, return_log_probs=True, finalize=fin)
        out, lp, att = dec.decode(enc, return_log_probs=True, return_attention=True, finalize=fin)
        assert torch.equal(out.ids, out0.ids) and torch.equal(lp, lp0)
        assert (att.sum(dim=3) - 1).abs().max().item() < 1e-4
