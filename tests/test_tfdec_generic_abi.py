"""CPU (-m "not gpu"): the generic-mode fields of lo_tfdec_args (upstream gradients of the TF-flavour decoder's logits and
alphas) are in the ctypes mirror after ``ws``, and lo_tfdec_backward validates them before it touches the device."""
import ctypes

from latex_ocr_b200 import tf_decoder


def test_tf_generic_backward_fields_and_validation_without_gpu():
    L = tf_decoder._bind()
    assert L.lo_sizeof_tfdec_args() == ctypes.sizeof(tf_decoder.TfDecArgs)
    names = [f[0] for f in tf_decoder.TfDecArgs._fields_]
    assert names[-4:] == ["ws", "dlogits_ext", "dlogits_stride", "dalpha_ext"]
    assert dict(tf_decoder.TfDecArgs._fields_)["dlogits_stride"] is ctypes.c_int64
    a = tf_decoder.TfDecArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.O, a.E, a.V = 2, 3, 8, 512, 256, 512, 512, 80, 40
    a.dt = 0
    # never dereferenced: the arguments are refused before any GPU work
    for k in ("enc", "ws", "logits", "alphas", "w_img", "w_cat2", "beta", "w_lstm", "b_lstm", "w_oc", "w_y", "w_init", "b_init", "emb",
              "formula", "denc", "g_w_img", "g_w_cat2", "g_beta", "g_w_lstm", "g_b_lstm", "g_w_oc", "g_w_y", "g_w_init", "g_b_init",
              "g_emb"):
        setattr(a, k, 0x1000)
    a.formula_stride = a.T
    a.dlogits_ext, a.dlogits_stride = 0x1000, a.V - 1
    assert L.lo_tfdec_backward(ctypes.byref(a), None) == -1
    assert b"dlogits_stride >= V" in L.lo_last_error()
    a.dlogits_ext, a.dlogits_stride, a.dalpha_ext = None, a.V, 0x1000
    assert L.lo_tfdec_backward(ctypes.byref(a), None) == -1
    assert b"dalpha_ext needs dlogits_ext" in L.lo_last_error()
