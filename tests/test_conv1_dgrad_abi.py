"""CPU (-m "not gpu"): lo_conv1_pool_dgrad_code (conv1's data gradient through the ReLU and the max-pool) refuses bad arguments
with a message before it touches the device."""
import pytest

from latex_ocr_b200 import _lib

P = 0x1000          # never dereferenced: every call below is refused before any GPU work


def _call(code=P, dpool=P, dt=_lib.LO_F32, w=P, dimg=P, N=2, H=32, W=64):
    L = _lib.lib()
    rc = L.lo_conv1_pool_dgrad_code(code, dpool, dt, w, 1.0, dimg, N, H, W, None)
    return rc, L.lo_last_error()


@pytest.mark.parametrize("which", ["code", "dpool", "w", "dimg"])
def test_null_pointers_are_refused(which):
    rc, msg = _call(**{which: None})
    assert rc == -1 and b"lo_conv1_pool_dgrad_code" in msg and b"null pointer" in msg, msg


@pytest.mark.parametrize("dt", [2, -1])
def test_bad_dtype_is_refused(dt):
    rc, msg = _call(dt=dt)
    assert rc == -1 and b"dt must be LO_F32 or LO_BF16" in msg, msg


@pytest.mark.parametrize("shape", [dict(N=0), dict(N=-3), dict(H=1), dict(W=1), dict(H=0, W=0)])
def test_bad_shape_is_refused(shape):
    rc, msg = _call(**shape)
    assert rc == -1 and b"shape (N >= 1, H >= 2, W >= 2)" in msg, msg
