"""-m gpu: decoding a list of images of different sizes in one time loop (lo_decoder_args.reg_off): every image attends over its
own regions only, so its tokens are those of the CPU oracle (oracle/ref_decode.py) decoding that image alone, and a batch of one
size gives the tensor path's results bit for bit."""
import pytest
import torch

from util import build_model

pytestmark = pytest.mark.gpu

V = 30


def _params(seed):
    """oracle parameters with a non-degenerate argmax: larger output layer and embedding (as in test_gpu_decode._setup)"""
    from oracle import ref_model as rm
    pe, pd = rm.init_params(V, seed=seed)
    g = torch.Generator().manual_seed(seed)
    pd["fc.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 0.5
    pd["embedding.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 1.0
    return pe, pd


def _mixed(seed, shapes=((32, 64), (48, 96), (32, 200), (48, 64), (32, 128)), per=2):
    """[1,H,W] float images of several shapes, interleaved so that no two neighbours share a shape"""
    from oracle import ref_model as rm
    groups = [rm.synthetic_batch(per, H, W, V, 3, 5, seed=seed + k)[0] for k, (H, W) in enumerate(shapes)]
    return [groups[k][i] for i in range(per) for k in range(len(shapes))]


def _enc(pe, img):
    from oracle import ref_model as rm
    return rm.encoder_forward(pe, img.unsqueeze(0)).reshape(1, -1, 512)


def test_greedy_mixed_sizes_match_the_oracle_per_image():
    from latex_ocr_b200 import decode
    from oracle import ref_decode as rd
    pe, pd = _params(4)
    m = build_model(V, pe, pd, "fp32")
    imgs = _mixed(10)
    for end_id, L in ((V - 1, 6), (7, 12), (3, 12)):
        got = decode.greedy_decode(m, imgs, start_id=V - 2, end_id=end_id, max_length_formula=L)
        wants = [rd.greedy_decode(pd, _enc(pe, x), start_id=V - 2, end_id=end_id, max_iter=L + 1)[0] for x in imgs]
        assert got.shape == (len(imgs), max(w.shape[0] for w in wants))
        for i, w in enumerate(wants):
            assert torch.equal(got[i, :w.shape[0]], w), (end_id, i)
    # the end ids above finish rows at different steps
    lens = {rd.greedy_decode(pd, _enc(pe, x), start_id=V - 2, end_id=7, max_iter=13).shape[1] for x in imgs}
    assert len(lens) > 1


@pytest.mark.parametrize("beam", [1, 3, 5])
def test_beam_mixed_sizes_match_the_oracle_per_image(beam):
    from latex_ocr_b200 import decode
    from oracle import ref_decode as rd
    pe, pd = _params(6)
    m = build_model(V, pe, pd, "fp32")
    imgs = _mixed(20, per=1)
    L = 8
    for fin in ("reference", "backtrack"):
        got, glp = decode.beam_decode(m, imgs, start_id=V - 2, end_id=5, beam_size=beam, max_length_formula=L, finalize=fin)
        for i, x in enumerate(imgs):
            want, wlp = rd.beam_decode(pd, _enc(pe, x), start_id=V - 2, end_id=5, beam=beam, max_iter=L + 1, finalize=fin)
            w = want[0].permute(1, 0)                               # [beam, steps_i]
            assert torch.equal(got[i, :, :w.shape[1]], w), (fin, i)
            assert (glp[i] - wlp[0]).abs().max().item() < 1e-3 * max(1.0, wlp.abs().max().item())
    # diversity penalty with injected uniforms: image i draws its rows [i*beam, (i+1)*beam)
    u = torch.rand(L + 2, len(imgs) * beam, V, generator=torch.Generator().manual_seed(77))
    got, glp = decode.beam_decode(m, imgs, start_id=V - 2, end_id=5, beam_size=beam, max_length_formula=L, div_gamma=0.5,
                                  div_prob=0.7, div_u=u)
    for i, x in enumerate(imgs):
        want, wlp = rd.beam_decode(pd, _enc(pe, x), start_id=V - 2, end_id=5, beam=beam, max_iter=L + 1, div_gamma=0.5, div_prob=0.7,
                                   div_u=u[:, i * beam:(i + 1) * beam])
        w = want[0].permute(1, 0)
        assert torch.equal(got[i, :, :w.shape[1]], w), i
        assert (glp[i] - wlp[0]).abs().max().item() < 1e-3 * max(1.0, wlp.abs().max().item())


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_uniform_sizes_through_the_list_reproduce_the_tensor_path_bit_for_bit(precision):
    """One image size (cfg #2: 128 x 512 px, R = 868): the ragged attention kernel partitions every row as the dense one does."""
    from latex_ocr_b200 import decode
    from oracle import ref_model as rm
    pe, pd = _params(8)
    m = build_model(V, pe, pd, precision, impl="tc" if precision == "bf16" else "simt")
    for N in (3, 40, 64):
        img, _ = rm.synthetic_batch(N, 128, 512, V, 3, 5, seed=30 + N)
        ids_t, al_t = decode.greedy_decode(m, img, V - 2, V - 1, 8, return_attention=True)
        ids_l, al_l = decode.greedy_decode(m, list(img), V - 2, V - 1, 8, return_attention=True)
        assert al_t.shape[2] == 868
        assert torch.equal(ids_t, ids_l), N
        assert torch.equal(al_t, torch.stack(al_l)), N
    img, _ = rm.synthetic_batch(8, 128, 512, V, 3, 5, seed=50)
    ids_t, lp_t = decode.beam_decode(m, img, V - 2, 5, 5, 8)
    ids_l, lp_l = decode.beam_decode(m, list(img), V - 2, 5, 5, 8)
    assert torch.equal(ids_t, ids_l) and torch.equal(lp_t, lp_l)


def test_attention_export_per_image():
    from latex_ocr_b200 import decode
    from oracle import ref_model as rm
    pe, pd = _params(4)
    m = build_model(V, pe, pd, "fp32")
    imgs = _mixed(40)
    ids, att = decode.greedy_decode(m, imgs, start_id=V - 2, end_id=V - 1, max_length_formula=6, return_attention=True)
    assert len(att) == len(imgs)
    for x, a in zip(imgs, att):
        h, w = m.encoder.out_hw(x.shape[1], x.shape[2])
        assert a.shape == (ids.shape[1], h * w)
        assert (a.sum(dim=1) - 1).abs().max().item() < 1e-4
        enc = _enc(pe, x)
        h0, _ = rm.init_hidden_state(pd, enc)
        _, a0 = rm.attention_forward(pd, enc, h0)
        assert (a[0] - a0[0]).abs().max().item() < 1e-5
        assert decode.attention_maps(a, h, w).shape == (ids.shape[1], h, w)


def _subset_alone_and_inside(m, decode, small, big):
    """tokens and alphas of `small` decoded alone and at their positions inside `big`"""
    ids_s, al_s = decode.greedy_decode(m, small, V - 2, V - 1, 10, return_attention=True)
    ids_b, al_b = decode.greedy_decode(m, big, V - 2, V - 1, 10, return_attention=True)
    return ids_s, al_s, ids_b, al_b


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_an_image_decodes_the_same_alone_and_in_any_composition(precision):
    from latex_ocr_b200 import _lib, decode
    pe, pd = _params(12)
    m = build_model(V, pe, pd, precision, impl="tc" if precision == "bf16" else "simt")
    small = _mixed(60, shapes=((32, 64), (48, 160)), per=2)
    extra = _mixed(70, per=5)                                                   # 25 more images of five shapes
    big = small + extra
    perm = torch.randperm(len(big), generator=torch.Generator().manual_seed(3)).tolist()
    big = [big[i] for i in perm]
    pos = [perm.index(i) for i in range(len(small))]
    if precision == "fp32":
        ids_s, al_s, ids_b, al_b = _subset_alone_and_inside(m, decode, small, big)
        n = ids_s.shape[1]
        assert torch.equal(ids_s, ids_b[pos, :n])
        for i, p in enumerate(pos):
            assert (al_s[i] - al_b[p][:n]).abs().max().item() < 1e-5
    # a fixed split count partitions every row the same whatever the composition: bit-identical (at most 64 rows)
    with _lib.option(att_nsplit=3):
        ids_s, al_s, ids_b, al_b = _subset_alone_and_inside(m, decode, small, big)
    n = ids_s.shape[1]
    assert torch.equal(ids_s, ids_b[pos, :n])
    for i, p in enumerate(pos):
        assert torch.equal(al_s[i], al_b[p][:n])


def test_predict_images_surface_and_workspace_reuse():
    pe, pd = _params(8)
    m = build_model(V, pe, pd, "fp32")
    imgs = [x.to(torch.uint8) for x in _mixed(80)]
    arrays = [x.permute(1, 2, 0).numpy() for x in imgs]                          # HxWx1 uint8 arrays
    for dec, k in (("greedy", 1), ("beam_search", 2)):
        out = m.predict_images(arrays, decoding=dec, beam_size=k)
        ref = m.predict_batch(arrays, decoding=dec, beam_size=k)
        assert len(out) == len(ref) == k and all(len(h) == len(imgs) for h in out)
        assert all(V - 1 not in seq for hyp in out for seq in hyp)           # truncated at END
    # tensors and arrays of the same images decode alike
    assert m.predict_images(imgs) == m.predict_images(arrays)
    # compositions that fit the first workspace reuse it
    m.predict_images(arrays)
    n = len(m.decoder._ws)
    m.predict_images(arrays[:3])
    m.predict_images(arrays[5:] + arrays[:2])
    assert len(m.decoder._ws) == n
