"""CPU (-m "not gpu"): lo_beam_backtrack, the hypotheses and their attention weights after a beam search of either decoder flavour.
The entry point is bound from the header, every bad argument is refused with LO_EINVAL before any GPU work, and the rule it
implements holds on the CPU oracles: under 'backtrack', the attention rows their beam search computes (recorded by
tests/beam_oracle.py), followed back along each hypothesis's lineage, are those of a teacher-forced pass over the hypothesis's own
tokens (both flavours, float64)."""
import ctypes

import pytest
import torch

import beam_oracle as bo
from latex_ocr_b200 import _lib

# never dereferenced: every call below is refused before any GPU work
_FAKE = 0x1000


@pytest.fixture
def L():
    return _lib.lib()


def test_bound_from_the_header(L):
    assert "lo_beam_backtrack" in _lib.declared_symbols()
    restype, argtypes = _lib.declared_signatures()["lo_beam_backtrack"]
    assert restype is ctypes.c_int and len(argtypes) == 15
    assert argtypes[2] is ctypes.c_int64 and argtypes[7] is ctypes.c_int64 and argtypes[11] is ctypes.c_int
    assert L.lo_beam_backtrack.argtypes == argtypes


def _call(L, off=None, **kw):
    """3 images, beam 2, n = 4 of 6 steps, R = 8; ``off``: host region offsets (the device ones are then a fake pointer)"""
    args = dict(ids=_FAKE, parents=_FAKE, stride=6, n_img=3, beam=2, n=4, alphas=_FAKE, row_stride=6 * 8, R=8, reg_off=None,
                reg_off_host=None, mode=_lib.LO_BEAM_LINEAGE, ids_out=_FAKE, att_out=_FAKE)
    if off is not None:
        host = (ctypes.c_int32 * len(off))(*off)
        args.update(reg_off=_FAKE, reg_off_host=ctypes.cast(host, ctypes.c_void_p).value)
    args.update(kw)
    rc = L.lo_beam_backtrack(*args.values(), None)
    return rc, L.lo_last_error()


BAD = [
    ({"ids": None}, b"null ids"),
    ({"parents": None}, b"null ids"),
    ({"ids_out": None}, b"null ids"),
    ({"alphas": None}, b"set together"),
    ({"att_out": None}, b"set together"),
    ({"beam": 0}, b"1 <= beam <= 16"),
    ({"beam": 17}, b"1 <= beam <= 16"),
    ({"n_img": 0}, b"n_img >= 1"),
    ({"n": 0}, b"1 <= n <= ids_stride_steps"),
    ({"n": 7}, b"1 <= n <= ids_stride_steps"),
    ({"mode": 2}, b"mode must be"),
    ({"mode": -1}, b"mode must be"),
    ({"R": 0, "row_stride": 0}, b"1 <= R"),
    ({"row_stride": 4 * 8 - 1}, b"alpha_row_stride >= n * R"),
    ({"reg_off": _FAKE}, b"reg_off and reg_off_host must be set together"),
    ({"stride": 4000, "n": 4000, "beam": 2, "row_stride": 4000 * 8}, b"48 kB"),
]


@pytest.mark.parametrize("kw,msg", BAD, ids=[m.decode() + "-" + ",".join(k) for k, m in BAD])
def test_bad_arguments_are_refused(L, kw, msg):
    rc, err = _call(L, **kw)
    assert rc == -1 and msg in err, err


@pytest.mark.parametrize("off", [[0, 2, 2, 8], [0, 3, 1, 4], [0, 9, 12, 14], [0, 1, 2, 11]])
def test_region_counts_outside_one_to_R_are_refused(L, off):
    rc, err = _call(L, off)
    assert rc == -1 and b"region count of every image in 1..R" in err


# ------------------------------------------------------------------------------------------------ the rule, on the CPU oracles
V = 30


def _enc(N, R, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.relu(torch.randn(N, R, 512, generator=g)) * 0.7).double()


def test_torch_oracle_backtracked_attention_is_the_teacher_forced_attention():
    from oracle import ref_decode as rd
    from oracle import ref_model as rm
    _, pd = rm.init_params(V, seed=3)
    g = torch.Generator().manual_seed(3)
    pd["fc.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 0.5
    pd["embedding.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 1.0
    pd = {k: v.double() for k, v in pd.items()}
    enc = _enc(3, 12, 5)
    beam = 4
    ids, lp, alphas, parents = bo.recorded_beam("torch", pd, enc, V, V - 2, 5, beam, 8, finalize="backtrack")
    assert (parents != torch.arange(beam)).any(), "the lineages must cross slots for the test to mean anything"
    hyps = ids.permute(0, 2, 1)
    att = bo.hypothesis_attention(alphas, parents, "backtrack")
    tf = bo.teacher_forced_attention(pd, enc, V - 2, hyps)
    assert (att - tf).abs().max().item() < 1e-12
    # the slot rows are not (the test distinguishes the two views) ...
    assert (bo.hypothesis_attention(alphas, parents, "reference") - tf).abs().max().item() > 1e-6
    # ... and recording leaves the oracle's results unchanged
    ids2, lp2 = rd.beam_decode(pd, enc, V - 2, 5, beam, 8, finalize="backtrack")
    assert torch.equal(ids, ids2) and torch.equal(lp, lp2)
    assert torch.equal(rd.backtrack(bo.recorded_beam("torch", pd, enc, V, V - 2, 5, beam, 8)[0], parents), ids)


def test_tf_oracle_backtracked_attention_is_the_teacher_forced_attention():
    from oracle import ref_decode as rd
    from oracle import ref_tf_model as tfm
    p = tfm.init_params_tf(V, seed=4, dtype=torch.float64)
    p["y_W_o"] = p["y_W_o"] * 4.0
    enc = _enc(3, 10, 6)
    beam = 3
    u = torch.rand(11, 3 * beam, V, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    for kw in ({}, {"div_gamma": 0.5, "div_prob": 0.7, "div_u": u}):
        ids, lp, alphas, parents = bo.recorded_beam("tf", p, enc, V, 5, beam, 9, **kw)
        assert (parents != torch.arange(beam)).any()
        hyps = rd.backtrack(ids, parents).permute(0, 2, 1)
        att = bo.hypothesis_attention(alphas, parents, "backtrack")
        tf = bo.tf_teacher_forced_attention(p, enc, hyps)
        assert (att - tf).abs().max().item() < 1e-12, kw
        ids2, lp2 = tfm.beam_decode(p, enc, 5, beam, 9, **kw)
        assert torch.equal(ids, ids2) and torch.equal(lp, lp2)
