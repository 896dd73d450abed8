"""CPU (-m "not gpu"): lo_attention_step_backward (the backward of one stand-alone Attention.forward call) refuses bad arguments
with a message before it touches the device, and its workspace size follows the documented regions."""
import pytest

from latex_ocr_b200 import _lib

P = 0x1000          # never dereferenced: every call below is refused before any GPU work
INPUTS = ("enc", "att1", "h", "att2", "w_enc", "w_dec", "wf", "alpha", "ctx", "dctx", "work")


def _call(dt=_lib.LO_BF16, B=4, R=44, A=512, C=512, D=512, impl=_lib.LO_IMPL_TC, **null):
    L = _lib.lib()
    p = {k: (None if k in null else P) for k in INPUTS}
    rc = L.lo_attention_step_backward(p["enc"], p["att1"], dt, p["h"], p["att2"], p["w_enc"], p["w_dec"], p["wf"], p["alpha"],
                                      p["ctx"], p["dctx"], None, *([P] * 8), None, None, None, B, R, A, C, D, impl, p["work"], None)
    return rc, L.lo_last_error()


@pytest.mark.parametrize("which", INPUTS)
def test_null_inputs_are_refused(which):
    rc, msg = _call(**{which: True})
    assert rc == -1 and b"lo_attention_step_backward" in msg and b"null pointer" in msg, msg


@pytest.mark.parametrize("dt", [2, -1])
def test_bad_dtype_is_refused(dt):
    rc, msg = _call(dt=dt)
    assert rc == -1 and b"dt must be LO_F32 or LO_BF16" in msg, msg


def test_bad_impl_is_refused():
    rc, msg = _call(impl=2)
    assert rc == -1 and b"impl must be LO_IMPL_SIMT or LO_IMPL_TC" in msg, msg


@pytest.mark.parametrize("AC", [(256, 512), (512, 256), (384, 384), (128, 128), (2048, 2048)])
def test_unsupported_widths_are_refused(AC):
    A, C = AC
    rc, msg = _call(A=A, C=C)
    assert rc == -1 and b"attention_dim == encoder_dim in {256,512,1024}" in msg, msg


@pytest.mark.parametrize("shape", [dict(B=0), dict(B=513), dict(B=-1), dict(R=0), dict(R=-5), dict(D=0)])
def test_bad_shape_is_refused(shape):
    rc, msg = _call(**shape)
    assert rc == -1 and b"B in 1..512, R > 0, D > 0" in msg, msg


@pytest.mark.parametrize("dt,es", [(_lib.LO_F32, 4), (_lib.LO_BF16, 2)])
def test_workspace_bytes(dt, es):
    L = _lib.lib()
    B, R, A, C = 64, 868, 512, 512

    def al(n):
        return (n + 255) // 256 * 256
    want = (al(L.lo_attention_workspace_bytes(B, C)) + 2 * al(B * A * 4) + al(B * R * 4) + al(B * 4) + al(B * R * A * es)
            + al(A * C * 2))
    assert L.lo_attention_step_workspace_bytes(B, R, A, C, dt) == want
    assert L.lo_attention_step_workspace_bytes(0, R, A, C, dt) == 0


@pytest.mark.parametrize("which", ["enc", "att1", "datt1"])
def test_misaligned_pointers_are_refused(which):
    L = _lib.lib()
    p = {"enc": P, "att1": P, "datt1": P}
    p[which] = P + 4
    rc = L.lo_attention_step_backward(p["enc"], p["att1"], _lib.LO_BF16, P, P, P, P, P, P, P, P, None, *([P] * 8), None, None,
                                      p["datt1"], 4, 44, 512, 512, 512, _lib.LO_IMPL_TC, P, None)
    msg = L.lo_last_error()
    assert rc == -1 and b"must be 16-byte aligned" in msg, msg
