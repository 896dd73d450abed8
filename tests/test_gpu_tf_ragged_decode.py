"""-m gpu: the TensorFlow-flavour decoder (Genthial cell) decoding a list of images of different sizes in one time loop
(lo_tfdec_args.reg_off): every image attends over its own regions only, so its ids are those of the CPU oracle
(oracle/ref_tf_model.py) decoding that image alone, and a list of one size gives the tensor path's results bit for bit."""
import pytest
import torch

from util import Cfg

pytestmark = pytest.mark.gpu

V = 40
# (H, W) feature maps of the encoder outputs in the mixed lists: five region counts
SHAPES = ((4, 8), (6, 12), (4, 25), (6, 8), (4, 16))


def _cfg(**kw):
    kw.setdefault("max_length_formula", 10)
    return Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, **kw)


def _params(seed):
    from oracle import ref_tf_model as tfm
    p = tfm.init_params_tf(V, seed=seed)
    p["y_W_o"] = p["y_W_o"] * 4.0                               # sharper logits: non-degenerate argmax / beams
    return p


def _decoder(p, end_id=V - 1, precision="fp32", **kw):
    from latex_ocr_b200.tf_decoder import Decoder
    dec = Decoder(_cfg(**kw), V, end_id, device="cuda", precision=precision, impl="tc" if precision == "bf16" else "simt")
    dec.load_tf_variables(p)
    return dec


def _mixed(seed, shapes=SHAPES, per=2):
    """CPU encoder outputs [H, W, 512] of several sizes, interleaved so that no two neighbours share a size"""
    g = torch.Generator().manual_seed(seed)
    groups = [[torch.relu(torch.randn(h, w, 512, generator=g)) * 0.7 for _ in range(per)] for h, w in shapes]
    return [groups[k][i] for i in range(per) for k in range(len(shapes))]


def _dev(encs):
    """to the device, alternately as [H, W, C] and as [R, C]"""
    return [e.cuda() if i % 2 == 0 else e.reshape(-1, 512).cuda() for i, e in enumerate(encs)]


def _one(e):
    return e.reshape(1, -1, 512)


def test_greedy_mixed_sizes_match_the_oracle_per_image():
    from oracle import ref_tf_model as tfm
    p = _params(5)
    encs = _mixed(10)
    # end ids the rows emit at different steps: image 0's token of step 1 and image 3's of step 4 under an end id never emitted
    first = _decoder(p, V - 1, decoding="greedy").decode(_dev(encs)).ids.cpu()
    lens = set()
    for end_id in (V - 1, int(first[0, 1]), int(first[3, 4])):
        dec = _decoder(p, end_id, decoding="greedy")
        got = dec.decode(_dev(encs)).ids.cpu()
        wants = [tfm.greedy_decode(p, _one(e), end_id=end_id, max_iter=dec.max_length_formula + 1)[0] for e in encs]
        assert got.shape == (len(encs), max(w.shape[0] for w in wants))
        for i, w in enumerate(wants):
            assert torch.equal(got[i, :w.shape[0]], w), (end_id, i)
        lens |= {w.shape[0] for w in wants}
    assert len(lens) > 1                                         # the end ids above finish rows at different steps


@pytest.mark.parametrize("beam", [1, 2, 5])
def test_beam_mixed_sizes_match_the_oracle_per_image(beam):
    from oracle import ref_tf_model as tfm
    p = _params(7)
    encs = _mixed(20, per=1)
    dec = _decoder(p, 5, decoding="beam_search", beam_size=beam)
    L = dec.max_length_formula
    out, lp = dec.decode(_dev(encs), return_log_probs=True)
    lp = lp.cpu()
    for i, e in enumerate(encs):
        want, wlp = tfm.beam_decode(p, _one(e), end_id=5, beam=beam, max_iter=L + 1)
        assert torch.equal(out.ids[i, :want.shape[1]].cpu(), want[0]), i
        assert (lp[i] - wlp[0]).abs().max().item() < 1e-3 * max(1.0, wlp.abs().max().item())
    # diversity penalty with injected uniforms: image i draws its rows [i*beam, (i+1)*beam)
    dec = _decoder(p, 5, decoding="beam_search", beam_size=beam, div_gamma=0.5, div_prob=0.7)
    u = torch.rand(L + 2, len(encs) * beam, V, generator=torch.Generator().manual_seed(77))
    out, lp = dec.decode(_dev(encs), div_u=u, return_log_probs=True)
    lp = lp.cpu()
    for i, e in enumerate(encs):
        want, wlp = tfm.beam_decode(p, _one(e), end_id=5, beam=beam, max_iter=L + 1, div_gamma=0.5, div_prob=0.7,
                                    div_u=u[:, i * beam:(i + 1) * beam])
        assert torch.equal(out.ids[i, :want.shape[1]].cpu(), want[0]), i
        assert (lp[i] - wlp[0]).abs().max().item() < 1e-3 * max(1.0, wlp.abs().max().item())


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_uniform_sizes_through_the_list_reproduce_the_tensor_path_bit_for_bit(precision):
    """One size (the 868 regions of a 128 x 512 px image): the ragged attention kernel partitions every row as the dense one does."""
    p = _params(8)
    g = torch.Generator().manual_seed(8)
    dec = _decoder(p, precision=precision, decoding="greedy")
    for N in (3, 40, 64):
        enc = (torch.relu(torch.randn(N, 868, 512, generator=g)) * 0.7).cuda()
        out_t, al_t = dec.decode(enc, return_attention=True)
        out_l, al_l = dec.decode(list(enc), return_attention=True)
        assert al_t.shape[2] == 868
        assert torch.equal(out_t.ids, out_l.ids), N
        assert torch.equal(al_t, torch.stack(al_l).cuda()), N
    dec = _decoder(p, 5, precision=precision, decoding="beam_search", beam_size=5)
    enc = (torch.relu(torch.randn(8, 868, 512, generator=g)) * 0.7).cuda()
    out_t, lp_t = dec.decode(enc, return_log_probs=True)
    out_l, lp_l = dec.decode(list(enc), return_log_probs=True)
    assert torch.equal(out_t.ids, out_l.ids) and torch.equal(lp_t, lp_l)


def test_attention_export_per_image():
    from oracle import ref_tf_model as tfm
    p = _params(5)
    encs = _mixed(40)
    dec = _decoder(p, decoding="greedy")
    out, att = dec.decode(_dev(encs), return_attention=True)
    assert len(att) == len(encs)
    for e, a in zip(encs, att):
        e1 = _one(e)
        assert a.shape == (out.ids.shape[1], e1.shape[1])
        assert (a.sum(dim=1) - 1).abs().max().item() < 1e-4
        c, h, o = tfm.initial_state(p, e1)
        _, _, a0 = tfm.cell_step(p, e1, e1 @ p["att_img.kernel"], p["start_token"].expand(1, -1), c, h, o)
        assert (a[0].cpu() - a0[0]).abs().max().item() < 1e-5


def _alone_and_inside(dec, small, big):
    out_s, al_s = dec.decode(_dev(small), return_attention=True)
    out_b, al_b = dec.decode(_dev(big), return_attention=True)
    return out_s.ids, al_s, out_b.ids, al_b


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_an_image_decodes_the_same_alone_and_in_any_composition(precision):
    from latex_ocr_b200 import _lib
    p = _params(12)
    dec = _decoder(p, precision=precision, decoding="greedy")
    small = _mixed(60, shapes=((4, 8), (6, 20)), per=2)
    big = small + _mixed(70, per=5)                               # 25 more of five sizes: 29 rows, under the 64 of mma.sync
    perm = torch.randperm(len(big), generator=torch.Generator().manual_seed(3)).tolist()
    big = [big[i] for i in perm]
    pos = [perm.index(i) for i in range(len(small))]
    if precision == "fp32":
        ids_s, al_s, ids_b, al_b = _alone_and_inside(dec, small, big)
        n = ids_s.shape[1]
        assert torch.equal(ids_s, ids_b[pos, :n])
        for i, q in enumerate(pos):
            assert (al_s[i] - al_b[q][:n]).abs().max().item() < 1e-5
    # a fixed split count partitions every row the same whatever the composition: bit-identical
    with _lib.option(att_nsplit=3):
        ids_s, al_s, ids_b, al_b = _alone_and_inside(dec, small, big)
    n = ids_s.shape[1]
    assert torch.equal(ids_s, ids_b[pos, :n])
    for i, q in enumerate(pos):
        assert torch.equal(al_s[i], al_b[q][:n])


def _model(**kw):
    from latex_ocr_b200.data import SimpleVocab
    from latex_ocr_b200.img2seq_tf import Img2SeqModel
    return Img2SeqModel(_cfg(**kw), vocab=SimpleVocab(V), device="cuda", precision="fp32").build_pred()


def _images(n, seed, sizes=((32, 64), (48, 96), (32, 200), (48, 64), (32, 128))):
    """uint8 [1,H,W] images of several sizes, interleaved"""
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (1,) + sizes[i % len(sizes)], generator=g, dtype=torch.uint8) for i in range(n)]


def test_predict_images_surface_and_workspace_reuse():
    imgs = _images(10, 80)
    arrays = [x.permute(1, 2, 0).numpy() for x in imgs]                        # HxWx1 uint8 arrays
    for dec, k in (("greedy", 1), ("beam_search", 2)):
        m = _model(decoding=dec, beam_size=k)
        out = m.predict_images(arrays)
        assert len(out) == k and all(len(h) == len(imgs) for h in out)
        assert all(m._vocab.id_end not in seq for hyp in out for seq in hyp)   # truncated at END
        assert m.predict_images(imgs) == out                                   # tensors and arrays of the same images alike
    # compositions that fit the first workspace reuse it
    n, ws = len(m.decoder._ws), m.decoder._ws["ragged"]["ws"].data_ptr()
    m.predict_images(arrays[:3])
    m.predict_images(arrays[5:] + arrays[:2])
    assert len(m.decoder._ws) == n and m.decoder._ws["ragged"]["ws"].data_ptr() == ws


def test_predict_images_over_512_rows_decodes_in_chunks():
    """103 images at beam 5 are 515 decoder rows, above the 512 of one call: two chunks in input order (102 + 1 images)"""
    from latex_ocr_b200 import _lib
    m = _model(decoding="beam_search", beam_size=5, max_length_formula=4)
    imgs = _images(103, 90, sizes=((32, 64), (32, 96)))
    with _lib.option(att_nsplit=2):
        whole = m.predict_images(imgs)
        parts = [m.predict_images(imgs[:102]), m.predict_images(imgs[102:])]
    assert len(whole) == 5 and all(len(h) == 103 for h in whole)
    assert whole == [a + b for a, b in zip(*parts)]
