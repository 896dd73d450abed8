"""-m gpu: the autograd node shared by the kernel-backed modules (latex_ocr_b200/kernel_module.py).  An output the loss does not
use gets no gradient pass: an unused ``alphas`` reaches lo_decoder_backward as ``dalpha_ext = NULL`` ("zero"), which must give the
bits explicit zeros give.  A backward reads the forward state its node holds, so it still runs, with the same bits, after a forward
of another shape evicted that state from the bounded workspace caches.  bf16 with the tensor-core kernels, option
``deterministic``."""
import pytest
import torch
import torch.nn.functional as F

from latex_ocr_b200 import _lib
from util import Cfg

pytestmark = pytest.mark.gpu

V = 50


def _row_model():
    """Encoder, decoder, row encoder, layer 2 and the two-layer decoder of the extension, random weights, eval mode."""
    from latex_ocr_b200.ext import Img2SeqRowModel
    torch.manual_seed(5)
    m = Img2SeqRowModel(Cfg(), n_tok=V, device="cuda", precision="bf16", impl="tc")
    m.build_train()
    m.train_mode(False)
    return m


def _enc(B, R, seed):
    return (torch.randn(B, R, 512, generator=torch.Generator().manual_seed(seed)) * 0.5).cuda()


def _captions(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    formula = torch.randint(0, V, (B, T + 1), generator=g).cuda()
    lengths = torch.randint(2, T + 2, (B, 1), generator=g)
    lengths[0, 0] = T + 1
    return formula, lengths


def _ce(preds, caps, decode_lengths):
    T = preds.shape[1]
    act = (torch.arange(T, device=preds.device)[None, :] < torch.tensor(decode_lengths, device=preds.device)[:, None]).float()
    nll = -F.log_softmax(preds, dim=-1).gather(2, caps[:, 1:T + 1].unsqueeze(2)).squeeze(2)
    return (nll * act).sum() / act.sum()


@pytest.mark.parametrize("two_layer", [False, True], ids=["DecoderWithAttention", "TwoLayerDecoder"])
def test_unused_alphas_give_the_bits_of_explicit_zeros(two_layer):
    m = _row_model()
    dec = m.decoder2 if two_layer else m.decoder
    enc = _enc(4, 12, seed=1)
    formula, lengths = _captions(4, 8, seed=2)

    def grads(zero_alphas_term):
        dec.zero_grad(set_to_none=True)
        x = enc.clone().requires_grad_(True)
        preds, caps, dl, alphas, _ = dec(x, formula, lengths)
        loss = _ce(preds, caps, dl)
        if zero_alphas_term:
            loss = loss + 0 * alphas.sum()             # d alphas arrives as explicit zeros
        loss.backward()
        return [x.grad] + [p.grad.clone() for p in dec.parameters()]

    with _lib.option(deterministic=1):
        unused, zeros = grads(False), grads(True)
    names = ["d encoder_out"] + [k for k, _ in dec.named_parameters()]
    for name, a, b in zip(names, unused, zeros):
        assert torch.equal(a, b), name


def _tf_decoder():
    from latex_ocr_b200.tf_decoder import Decoder
    torch.manual_seed(6)
    cfg = Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=10)
    return Decoder(cfg, V, V - 1, device="cuda", precision="bf16", impl="tc")


def _cases():
    """name -> (module, its workspace caches, forward A -> (scalar loss, inputs whose gradients to compare), a forward of another
    shape)."""
    m = _row_model()
    tf = _tf_decoder()
    g = torch.Generator().manual_seed(7)
    img_a, img_b = (torch.rand(2, 1, 32, 64, generator=g) * 255).cuda(), (torch.rand(3, 1, 32, 96, generator=g) * 255).cuda()
    feat_a, feat_b = _enc(2, 12, seed=8).view(2, 2, 6, 512), _enc(3, 5, seed=9).view(3, 1, 5, 512)
    enc_a, enc_b = _enc(4, 12, seed=10), _enc(3, 9, seed=11)
    (f_a, l_a), (f_b, l_b) = _captions(4, 8, seed=12), _captions(3, 5, seed=13)
    # TF decoder: one row of distinct tokens, because its embedding-table gradient is scattered with fp32 atomics whose order
    # option deterministic does not fix (two identical backwards differ in the last bits when a token row is hit twice)
    tf_enc_a, tf_a = _enc(1, 12, seed=19), torch.randperm(V, generator=g)[:7].view(1, 7).cuda()
    tf_b = torch.randint(0, V, (3, 5), generator=g).cuda()

    def weighted(out, seed):
        return (out * torch.randn(out.shape, generator=torch.Generator().manual_seed(seed)).cuda()).sum()

    def encoder_a():
        x = img_a.clone().requires_grad_(True)
        return weighted(m.encoder(x), 14), [x]

    def row_encoder_a():
        x = feat_a.clone().requires_grad_(True)
        return weighted(m.row_encoder(x), 15), [x]

    def decoder_a(dec):
        def run():
            x = enc_a.clone().requires_grad_(True)
            preds, caps, dl, alphas, _ = dec(x, f_a, l_a)
            return _ce(preds, caps, dl) + weighted(alphas, 16), [x]
        return run

    def tf_a_run():
        x = tf_enc_a.clone().requires_grad_(True)
        logits, alphas = tf.train_outputs(x, tf_a)
        return weighted(logits, 17) + weighted(alphas, 18), [x]

    return {
        "EncoderCNN": (m.encoder, [m.encoder._ws], encoder_a, lambda: m.encoder(img_b)),
        "DecoderWithAttention": (m.decoder, [m.decoder._ws], decoder_a(m.decoder), lambda: m.decoder(enc_b, f_b, l_b)),
        "tf_decoder.Decoder": (tf, [tf._ws], tf_a_run, lambda: tf.train_outputs(enc_b, tf_b)),
        "RowEncoder": (m.row_encoder, [m.row_encoder._out] + [d._ws for d in m.row_encoder.dirs], row_encoder_a,
                       lambda: m.row_encoder(feat_b)),
        "TwoLayerDecoder": (m.decoder2, [m.decoder._ws, m.layer2._x, m.layer2.dir._ws], decoder_a(m.decoder2),
                            lambda: m.decoder2(enc_b, f_b, l_b)),
    }


@pytest.mark.parametrize("name", ["EncoderCNN", "DecoderWithAttention", "tf_decoder.Decoder", "RowEncoder", "TwoLayerDecoder"])
def test_backward_after_eviction_gives_the_same_bits(name):
    module, caches, forward_a, forward_b = _cases()[name]
    for c in caches:
        c.maxsize = 1

    def run(evict):
        module.zero_grad(set_to_none=True)
        loss, inputs = forward_a()
        if evict:
            keys = [list(c.keys()) for c in caches]
            with torch.no_grad():
                forward_b()
            assert all(list(c.keys()) != k for c, k in zip(caches, keys)), "the later forward did not evict"
        loss.backward()
        return [x.grad for x in inputs] + [p.grad.clone() for p in module.parameters()]

    with _lib.option(deterministic=1):
        want, got = run(False), run(True)
    names = ["d input"] + [k for k, _ in module.named_parameters()]
    for k, a, b in zip(names, want, got):
        assert torch.equal(a, b), k
