"""CPU (-m "not gpu"): the bf16-shadow rule of FlatStore on kernel-backed modules built on the host (the shadow is re-cast from the
fp32 master exactly when the master changed since the last cast), and the size checks of the three argument-struct mirrors."""
import ctypes

import pytest
import torch

from latex_ocr_b200 import _lib
from util import Cfg

POISON = 12288.0          # exactly representable in bf16, far from any initial weight


def _encoder():
    from latex_ocr_b200.encoder import EncoderCNN
    return EncoderCNN(Cfg(), device="cpu", precision="bf16")


def _tf_decoder():
    from latex_ocr_b200.tf_decoder import Decoder
    return Decoder(Cfg(attn_cell_config={"num_units": 64, "dim_e": 32, "dim_o": 64, "dim_embeddings": 16}), 21, 20,
                   device="cpu", precision="bf16", channels=64)


def _recasts(S):
    """Poison the shadow, do what every forward does first, and report whether the shadow was re-cast from the master."""
    S.shadow.fill_(POISON)
    S.refresh_shadow()
    if torch.equal(S.shadow, S.master.to(torch.bfloat16)):
        return True
    assert bool((S.shadow == POISON).all())
    return False


@pytest.mark.parametrize("make", [_encoder, _tf_decoder], ids=["EncoderCNN", "tf_decoder.Decoder"])
def test_shadow_is_recast_exactly_when_the_master_changed(make):
    m = make()
    S = m.store
    p = next(iter(m.parameters()))
    assert _recasts(S)                                   # first use
    assert not _recasts(S)                               # no edit since: the (poisoned) shadow is kept
    with torch.no_grad():
        p.mul_(0.5)
    assert _recasts(S) and not _recasts(S)
    m.load_state_dict(make().state_dict())
    assert _recasts(S) and not _recasts(S)
    S.grad.fill_(1.0)
    opt = torch.optim.Adam(m.parameters(), lr=0.1)
    opt.step()
    assert _recasts(S) and not _recasts(S)
    with torch.no_grad():
        p.add_(1.0)
    S.shadow.fill_(POISON)
    S.mark_shadow_current()                              # master and shadow restored together: the shadow stands
    S.refresh_shadow()
    assert bool((S.shadow == POISON).all())
    S.sync_shadow()                                      # the unconditional cast still casts
    assert torch.equal(S.shadow, S.master.to(torch.bfloat16))


def test_struct_mirrors_match_the_library():
    L = _lib.lib()                                       # refuses to load on a size mismatch
    assert L.lo_sizeof_decoder_args() == ctypes.sizeof(_lib.DecoderArgs)
    assert L.lo_sizeof_tfdec_args() == ctypes.sizeof(_lib.TfDecArgs)
    assert L.lo_sizeof_lstm_seq_args() == ctypes.sizeof(_lib.LstmSeqArgs)
    from latex_ocr_b200 import ext, tf_decoder
    assert tf_decoder.TfDecArgs is _lib.TfDecArgs and ext.LstmSeqArgs is _lib.LstmSeqArgs
