"""-m gpu: the TensorFlow-flavour decoder (Genthial cell, SURVEY §8-a row a7) through the C ABI against the CPU restatement
oracle/ref_tf_model.py (parity UNPINNED: the reference runs this flavour only as a TF 1.12 graph, see the oracle's header).
fp32 mode: logits / loss / every gradient to 1e-4 of the tensor's max, token ids exact; bf16 mode: stated looser tolerances."""
import pytest
import torch

from util import Cfg, relerr

pytestmark = pytest.mark.gpu


def _cfg(**kw):
    return Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=10, **kw)


def _setup(V=40, N=3, R=21, T=7, seed=3, precision="fp32", impl="simt", **kw):
    from latex_ocr_b200.tf_decoder import Decoder
    from oracle import ref_tf_model as tfm
    g = torch.Generator().manual_seed(seed)
    p = tfm.init_params_tf(V, seed=seed)
    p["y_W_o"] = p["y_W_o"] * 4.0                               # sharper logits: non-degenerate argmax / beams
    enc = torch.relu(torch.randn(N, R, 512, generator=g)) * 0.7
    formula = torch.randint(0, V, (N, T), generator=g)
    dec = Decoder(_cfg(**kw), V, V - 1, device="cuda", precision=precision, impl=impl)
    dec.load_tf_variables(p)
    return tfm, p, dec, enc, formula


def _oracle_grads(tfm, p, enc, formula, lengths, keep_h=None, keep_o=None):
    p = {k: v.clone().double().requires_grad_(True) for k, v in p.items()}
    enc = enc.clone().double().requires_grad_(True)
    kh = None if keep_h is None else keep_h.double()
    ko = None if keep_o is None else keep_o.double()
    logits, alphas = tfm.decoder_train_logits(p, enc, formula, kh, ko)
    loss, ce_words, n_words = tfm.masked_ce(logits, formula, lengths)
    loss.backward()
    return logits.detach(), alphas.detach(), loss.detach(), {k: v.grad for k, v in p.items()}, enc.grad


@pytest.mark.parametrize("dropout", [False, True])
def test_tf_decoder_fp32_matches_oracle(dropout):
    tfm, p, dec, enc, formula = _setup()
    N, T = formula.shape
    lengths = torch.tensor([7, 5, 3])
    kh = ko = None
    if dropout:
        g = torch.Generator().manual_seed(11)
        kh = (torch.rand(N, T, 512, generator=g) < 0.8).float() / 0.8
        ko = (torch.rand(N, T, 512, generator=g) < 0.8).float() / 0.8
    logits, alphas, loss, grads, denc = _oracle_grads(tfm, p, enc, formula, lengths, kh, ko)
    got = dec.train_logits(enc.cuda(), formula.cuda(), kh, ko)
    assert got.shape == logits.shape
    assert relerr(got, logits) < 1e-4
    l, de = dec.loss_and_backward(enc.cuda(), formula.cuda(), lengths, kh, ko)
    torch.cuda.synchronize()
    assert abs(l[0].item() - loss.item()) / abs(loss.item()) < 1e-5
    assert abs(l[3].item() - float(lengths.sum())) < 1e-3
    ws = dec._ws[(N, T, enc.shape[1], 1)]
    assert relerr(ws["alphas"], alphas) < 1e-4
    assert relerr(de, denc) < 1e-4
    for k, q in dec.named_parameters():
        assert relerr(q.grad, grads[k].reshape(q.grad.shape)) < 1e-4, k


def test_tf_decoder_bf16_close_to_oracle():
    """bf16 storage / fp32 accumulate, wgmma + mma.sync GEMMs, tanh.approx in the attention score: loss within 2e-2 relative,
    gradients within 6e-2 of their max."""
    tfm, p, dec, enc, formula = _setup(N=4, R=40, T=9, precision="bf16", impl="tc")
    lengths = torch.tensor([9, 9, 6, 2])
    logits, alphas, loss, grads, denc = _oracle_grads(tfm, p, enc, formula, lengths)
    l, de = dec.loss_and_backward(enc.cuda(), formula.cuda(), lengths)
    torch.cuda.synchronize()
    assert abs(l[0].item() - loss.item()) / abs(loss.item()) < 2e-2
    assert relerr(de, denc) < 6e-2
    for k, q in dec.named_parameters():
        assert relerr(q.grad, grads[k].reshape(q.grad.shape)) < 6e-2, k


def test_tf_greedy_ids_match_oracle():
    tfm, p, dec, enc, formula = _setup(seed=5, decoding="greedy")
    want = tfm.greedy_decode(p, enc, end_id=dec._id_end, max_iter=dec.max_length_formula + 1)
    out = dec.decode(enc.cuda())
    assert out.ids.shape == want.shape, (out.ids.shape, want.shape)
    assert torch.equal(out.ids.cpu(), want)
    train, test = dec(enc.cuda(), formula.cuda(), 1.0)              # Decoder.__call__ surface: (pred_train, pred_test)
    assert train.shape == (formula.shape[0], formula.shape[1], 40) and torch.equal(test.ids.cpu(), want)


@pytest.mark.parametrize("beam", [2, 5])
def test_tf_beam_ids_match_oracle(beam):
    tfm, p, dec, enc, formula = _setup(seed=7, decoding="beam_search", beam_size=beam)
    want, wlp = tfm.beam_decode(p, enc, end_id=dec._id_end, beam=beam, max_iter=dec.max_length_formula + 1)
    out = dec.decode(enc.cuda())
    assert out.ids.shape == want.shape, (out.ids.shape, want.shape)
    assert torch.equal(out.ids.cpu(), want)


def test_tf_beam_diversity_penalty_and_attention_export():
    """div_gamma / div_prob of configs/model.json:15-16 switched on (beam_search_decoder_cell.py:258-287) with injected Bernoulli
    draws; greedy attention export (attention_mechanism.py:96-121)."""
    beam = 3
    tfm, p, dec, enc, formula = _setup(seed=7, decoding="beam_search", beam_size=beam, div_gamma=0.6, div_prob=0.7)
    steps = dec.max_length_formula + 2
    u = torch.rand(steps, enc.shape[0] * beam, 40, generator=torch.Generator().manual_seed(5))
    want, _ = tfm.beam_decode(p, enc, end_id=dec._id_end, beam=beam, max_iter=dec.max_length_formula + 1, div_gamma=0.6, div_prob=0.7,
                              div_u=u)
    out = dec.decode(enc.cuda(), div_u=u)
    assert out.ids.shape == want.shape and torch.equal(out.ids.cpu(), want)
    out2 = dec.decode(enc.cuda())                                   # in-kernel Philox draws
    assert out2.ids.shape[0] == enc.shape[0]
    tfm, p, dec, enc, formula = _setup(seed=5, decoding="greedy")
    out, att = dec.decode(enc.cuda(), return_attention=True)
    assert att.shape == (enc.shape[0], out.ids.shape[1], enc.shape[1])
    att_img = enc @ p["att_img.kernel"]
    c, h, o = tfm.initial_state(p, enc)
    _, _, a0 = tfm.cell_step(p, enc, att_img, p["start_token"].expand(enc.shape[0], -1), c, h, o)
    assert (att[:, 0].cpu() - a0).abs().max().item() < 1e-5


def test_tf_encoder_input_normalisation():
    """input_norm='tf': conv1 consumes (img - 128) / 128 (model/encoder.py:26-27) — against the oracle encoder on the normalised
    image; uint8 and float inputs agree bit for bit."""
    from latex_ocr_b200.encoder import EncoderCNN
    from oracle import ref_model as rm
    pe, _ = rm.init_params(20, seed=9)
    img, _ = rm.synthetic_batch(2, 32, 64, 20, 3, 4, seed=10)
    want = rm.encoder_forward(pe, (img - 128.0) / 128.0)
    enc = EncoderCNN(Cfg(input_norm="tf"), device="cuda", precision="fp32")
    enc.load_state_dict(pe)
    got = enc(img.cuda())
    got8 = enc(img.to(torch.uint8).cuda())
    assert relerr(got, want) < 1e-4
    assert torch.equal(got, got8)


def test_tf_model_trains_and_predicts():
    """TF-flavour Img2SeqModel surface: _run_train (one epoch over lists of HWC uint8 arrays + id lists), evaluate (negated
    perplexity), predict_batch (hypotheses x images); repeated steps on one batch reduce the loss."""
    import numpy as np
    from latex_ocr_b200.data import SimpleVocab
    from latex_ocr_b200.img2seq_tf import Img2SeqModel
    from latex_ocr_b200.lr_schedule import LRSchedule
    rng = np.random.RandomState(1)
    V = 30
    vocab = SimpleVocab(V)
    data = [(rng.randint(0, 256, (32, 64, 1)).astype(np.uint8), list(rng.randint(0, V - 3, 3 + i % 3))) for i in range(6)]
    cfg = _cfg(batch_size=3, n_epochs=1, decoding="beam_search", beam_size=2, dropout=1.0, lr_init=1e-3)
    m = Img2SeqModel(cfg, vocab=vocab, device="cuda", precision="fp32").build_train(cfg)
    score = m._run_train(cfg, data, data, 0, LRSchedule(lr_init=1e-3))
    assert score < 0 and np.isfinite(score)
    assert {"BLEU-4", "ExactMatchScore", "EditDistance", "perplexity", "images_per_s"} <= set(m.last_epoch_stats)
    imgs = [d[0] for d in data[:3]]
    forms = [d[1] for d in data[:3]]
    first = float(m.train_step(imgs, forms)[0])
    for _ in range(15):
        last = float(m.train_step(imgs, forms)[0])
    assert last < 0.7 * first, (first, last)
    hyps = m.predict_batch(imgs)
    assert len(hyps) == 2 and all(len(h) == 3 for h in hyps)
    assert all(vocab.id_end not in seq for seq in hyps[0])


@pytest.mark.parametrize("method,lr", [("sgd", 0.02), ("adagrad", 0.01), ("rmsprop", 1e-3)])
def test_tf_model_other_optimisers_reduce_the_loss(method, lr):
    """img2seq.py:98-111 offers adagrad / sgd / rmsprop besides adam; with clip_by_global_norm (:116-121) switched on."""
    import numpy as np
    from latex_ocr_b200.data import SimpleVocab
    from latex_ocr_b200.img2seq_tf import Img2SeqModel
    rng = np.random.RandomState(2)
    V = 30
    data = [(rng.randint(0, 256, (32, 64, 1)).astype(np.uint8), list(rng.randint(0, V - 3, 3 + i % 3))) for i in range(3)]
    cfg = _cfg(batch_size=3, n_epochs=1, decoding="greedy", dropout=1.0, lr_init=lr, lr_method=method, clip=5.0)
    m = Img2SeqModel(cfg, vocab=SimpleVocab(V), device="cuda", precision="fp32").build_train(cfg)
    imgs, forms = [d[0] for d in data], [d[1] for d in data]
    first = float(m.train_step(imgs, forms)[0])
    for _ in range(40):
        last = float(m.train_step(imgs, forms)[0])
    assert np.isfinite(last) and last < first, (method, first, last)        # the update rules themselves: test_gpu_kernels.py
    with pytest.raises(NotImplementedError):
        Img2SeqModel(_cfg(lr_method="lbfgs"), vocab=SimpleVocab(V), device="cuda", precision="fp32").build_train()
