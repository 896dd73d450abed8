"""-m gpu: the sequence LSTM (lo_lstm_seq_forward / lo_lstm_seq_backward, csrc/lo_lstmseq.cuh) launch by launch against float64,
under every schedule of its GEMMs, on the operands and layouts of its callers (RowEncoder's two directions, DecoderLayer2).

Each case calls the C ABI directly, from workspace views, outputs and gradient buffers filled with a finite sentinel, then
rebuilds every stored quantity in float64 (tests/lstmseq_step_ref.py) from the operands that launch read: the previous slot's
h_bf mirror (bf16 storage; h in fp32), dG_bf for the carried product and the hoisted GEMMs (dG in fp32), and the weights as the
kernels see them (the bf16 shadows in bf16, fp32 otherwise; the biases fp32).  So an error never compounds across steps.

Bounds: those derived in the docstring of tests/test_gpu_decoder_steps.py, with the same helpers (tests/step_check.py):
  * GEMM and reduction outputs (the pre-activations, the carried d h, the final dh, every weight gradient, the bias column sum,
    dxt): |y - ref| <= 2^-16 S, S the float64 sum of the magnitudes of the terms.
  * gates: their Lipschitz factor (1/4 for sigmoid, 1 for tanh) times the pre-activation allowance, plus 2^-21.
  * c and h from the kernel's own gates and c: 2^-22 (|f c_prev| + |i g|) and 2^-21 |h|.
  * d gates: dc is carried in float64 beside the kernel's fp32 chain, with its allowance E_dc; dh = dhs + carried gets the
    GEMM allowance of the carried product plus one rounding.
  * Exact: xt is the gather of x; bsum = fl(b_ih + b_hh); slot 0 holds h0 and c0 (or zeros); h_bf = RN(h) and dG_bf = RN(dG);
    whhT and wihT are the transposed weights; hs / hs_st hold h / RN(h) at time t(p), and the other direction's half of an
    interleaved output keeps the sentinel; g_b_hh = g_b_ih; dx is dxt scattered, or fl(base + dxt) with dx_accumulate; dh0 and
    dc0 are the final dh and dc; without dhs and h0 every gradient is 0.  The forward leaves the backward's views untouched.

Worst |y - ref| / bound per quantity, over every case and schedule, measured on an H100 80GB HBM3 (700 W power limit); the
whole file (35 tests) ran in 13 s there:
    pointwise: c 0.482, h 0.504, gates 0.013, dG 0.423, dc 0.024
    GEMMs and reductions (2^-16 S): dh 0.029, dxt 0.031, g_w_hh 0.038, g_w_ih 0.025, g_b 0.011
"""
import ctypes
from types import SimpleNamespace

import pytest
import torch

import lstmseq_step_ref as lr
from step_check import ACC, SENTINEL, Checker, cell_backward_bounds, check_cell, check_gates

pytestmark = pytest.mark.gpu


def _row_shape():
    """(H', W') of the feature map of a 160 x 640 image, by EncoderCNN's own arithmetic."""
    from latex_ocr_b200 import encoder
    return encoder.EncoderCNN.out_hw(SimpleNamespace(layers=encoder._LAYERS), 160, 640)


# name: (precision, impl, layout, S, M, I, H, options)
#   layout "row":   RowEncoder's two directions over a [N][H'][W'][C] map (M = N H', S = W'), interleaved bf16 output, the
#                   second direction's d x added onto the first's (M given as N; S and M follow from _row_shape)
#   layout "l2":    DecoderLayer2: x [B][T][D] in storage dtype, hs fp32 [B][T][D], d x written over d hs (the same buffer)
#   layout "plain": batch-major [M][S][I] with hs fp32 and hs_st, separate d x
#   options: "h0" (non-zero h0 / c0, dh0 / dc0 requested), "reverse", "nograd" (dhs = NULL)
_CASES = {
    "row2": ("bf16", "tc", "row", None, 2, 512, 256, ()),                # M = 36: mma.sync per-step GEMMs
    "row8": ("bf16", "tc", "row", None, 8, 512, 256, ()),                # M = 144: wgmma
    "l2b8": ("bf16", "tc", "l2", 7, 8, 512, 512, ()),                    # the carried product: K = 2048 in 4 K slices
    "l2b72": ("bf16", "tc", "l2", 7, 72, 512, 512, ()),
    "m1": ("bf16", "tc", "plain", 4, 1, 64, 128, ("reverse",)),
    "m64": ("bf16", "tc", "plain", 4, 64, 64, 128, ()),
    "m65": ("bf16", "tc", "plain", 4, 65, 64, 128, ("reverse",)),
    "h80m40": ("bf16", "tc", "plain", 5, 40, 48, 80, ("reverse",)),      # H % 64 != 0: no wgmma for the per-step product
    "h80m520": ("bf16", "tc", "plain", 5, 520, 48, 80, ()),              # above 512 rows: the CUDA-core bf16 product
    "init": ("bf16", "tc", "plain", 6, 48, 128, 128, ("h0", "reverse")),
    "nograd": ("bf16", "tc", "plain", 3, 16, 64, 64, ("nograd",)),
    "l2fp32": ("fp32", "simt", "l2", 7, 8, 512, 512, ()),                # fp32 dh product: K = 2048 split onto a zeroed C
    "bf16simt": ("bf16", "simt", "plain", 6, 24, 128, 64, ("h0",)),
}

# schedule -> (library options, the cases it runs)
_SCHEDULES = {
    "default": ({}, list(_CASES)),
    "skinny_mma0": ({"skinny_mma": 0}, ["row2", "l2b8", "m1", "m64", "h80m40"]),
    "skinny_tma0": ({"skinny_tma": 0}, ["row2", "l2b8", "m64"]),
    "skinny8_0": ({"skinny8": 0}, ["l2b72", "m65"]),
    "wgrad256": ({"wgrad256": 1}, ["row8", "l2b72"]),
    "pdl0": ({"pdl": 0}, ["row2", "l2b8", "l2b72"]),
    "deterministic": ({"deterministic": 1}, ["l2b8", "l2b72", "m64", "m65", "l2fp32", "h80m520"]),
}
_PARAMS = [(s, c) for s, (_, cs) in _SCHEDULES.items() for c in cs]

_WORST = {}


class _Dir:
    """One direction: weights, argument block and sentinel-filled workspace of shape (S, M, I, H)."""

    def __init__(self, precision, impl, S, M, I, H, reverse, h0, g):
        from latex_ocr_b200 import _lib
        self.bf = precision == "bf16"
        self.dt = torch.bfloat16 if self.bf else torch.float32
        self.S, self.M, self.I, self.H, self.reverse = S, M, I, H, reverse
        b = 1.0 / H ** 0.5

        def U(*shape):
            return ((torch.rand(*shape, device="cuda", generator=g) * 2 - 1) * b)
        self.w_ih, self.w_hh = U(4 * H, I).to(self.dt), U(4 * H, H).to(self.dt)
        self.b_ih, self.b_hh = U(4 * H), U(4 * H)
        self.h0 = self.c0 = self.dh0 = self.dc0 = None
        if h0:
            self.h0 = 0.5 * torch.randn(M, H, device="cuda", generator=g)
            self.c0 = torch.randn(M, H, device="cuda", generator=g)
            self.dh0 = torch.full((M, H), SENTINEL, device="cuda")
            self.dc0 = torch.full((M, H), SENTINEL, device="cuda")
        self.grads = {k: torch.full(s, SENTINEL, device="cuda") for k, s in
                      (("g_w_ih", (4 * H, I)), ("g_w_hh", (4 * H, H)), ("g_b_ih", (4 * H,)), ("g_b_hh", (4 * H,)))}
        a = self.a = _lib.LstmSeqArgs()
        a.S, a.M, a.I, a.H = S, M, I, H
        a.dt = _lib.dtype_code(precision)
        a.impl = _lib.impl_code(impl, precision)
        a.reverse = 1 if reverse else 0
        nbytes = int(_lib.lib().lo_lstm_seq_workspace_bytes(ctypes.byref(a)))
        self.ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")     # the padding between views compares equal
        self.v = lr.views(self.ws, S, M, I, H, self.bf)
        a.ws = self.ws.data_ptr()
        a.w_ih, a.w_hh, a.b_ih, a.b_hh = self.w_ih.data_ptr(), self.w_hh.data_ptr(), self.b_ih.data_ptr(), self.b_hh.data_ptr()
        for k in ("h0", "c0", "dh0", "dc0"):
            setattr(a, k, getattr(self, k).data_ptr() if getattr(self, k) is not None else None)
        for k, t in self.grads.items():
            setattr(a, k, t.data_ptr())

    def fill(self):
        for t in self.v.values():
            t.fill_(SENTINEL)
        for t in self.grads.values():
            t.fill_(SENTINEL)
        for t in (self.dh0, self.dc0):
            if t is not None:
                t.fill_(SENTINEL)

    def forward(self):
        from latex_ocr_b200 import _lib
        _lib.check(_lib.lib().lo_lstm_seq_forward(ctypes.byref(self.a), _lib.stream_ptr()))

    def backward(self):
        from latex_ocr_b200 import _lib
        _lib.check(_lib.lib().lo_lstm_seq_backward(ctypes.byref(self.a), _lib.stream_ptr()))

    def outputs(self):
        """Everything the calls write that lives in this direction's own buffers."""
        return [self.ws.clone()] + [t.clone() for t in self.grads.values()] + [t.clone() for t in (self.dh0, self.dc0) if t is not None]


def _strided(buf, off, M, S, n, row, step):
    """The [M][S][n] view of the elements (m, t) at off + m row + t step of a flat buffer."""
    return torch.as_strided(buf, (M, S, n), (row, step, 1), off)


def check_forward(ck, d, x, hs=None, hs_st=None, before_backward=True):
    """Every quantity the forward stored: x, hs, hs_st are the [M][S][.] views of the caller's tensors.  ``before_backward``:
    also that the backward's views still hold the sentinel."""
    v, S, H = d.v, d.S, d.H
    ts = lr.order(S, d.reverse)
    ck.exact("xt", v["xt"], lr.gather(x, d.reverse).to(d.dt))
    bsum = d.b_ih + d.b_hh                                                   # one fp32 addition
    ck.exact("bsum", v["bsum"], bsum)
    zero = torch.zeros(d.M, H, device="cuda")
    ck.exact("h slot 0", v["h"][0], d.h0 if d.h0 is not None else zero)
    ck.exact("c slot 0", v["c"][0], d.c0 if d.c0 is not None else zero)
    if d.bf:
        ck.exact("h_bf", v["h_bf"], v["h"].bfloat16())
    # the pre-activations: the hoisted product (+ bsum) plus the recurrent product of the mirror of slot p
    w_ih, w_hh = d.w_ih.double(), d.w_hh.double()
    hp = (v["h_bf"] if d.bf else v["h"])[:S].double()
    p_x, s_x = lr.input_projection(v["xt"].double(), w_ih, torch.zeros_like(bsum.double()), bsum.double())
    p_h, s_h = lr.recurrent(hp, w_hh)
    gates = v["gates"]
    check_gates(ck, gates, p_x + p_h, ACC * (s_x + s_h))
    i, f, g, o = gates.double().chunk(4, -1)
    check_cell(ck, v["c"][1:], v["h"][1:], i, f, g, o, v["c"][:S].double())
    if hs is not None:
        ck.exact("hs", hs[:, ts], v["h"][1:].transpose(0, 1))
    if hs_st is not None:
        ck.exact("hs_st", hs_st[:, ts], v["h"][1:].transpose(0, 1).to(hs_st.dtype))
    for k in ("dG", "dG_bf", "dh", "dc", "dxt", "whhT", "wihT") if before_backward else ():
        if k in v:
            ck.value("%s untouched by the forward" % k, v[k], SENTINEL)


def check_backward(ck, d, dhs, dx=None, base=None):
    """Every quantity the backward stored: dhs the [M][S][H] view of d hs as it was before the call (None: NULL), dx the view of
    the caller's d x, base what it held before the call (dx_accumulate) or None."""
    v, S, M, H = d.v, d.S, d.M, d.H
    ts = lr.order(S, d.reverse)
    ck.exact("whhT", v["whhT"], d.w_hh.t())
    ck.exact("wihT", v["wihT"], d.w_ih.t())
    w_ih, w_hh = d.w_ih.double(), d.w_hh.double()
    dG = v["dG"]
    if d.bf:
        ck.exact("dG_bf", v["dG_bf"], dG.bfloat16())
    dGa = (v["dG_bf"] if d.bf else dG).double()                              # what the carried and hoisted GEMMs read
    car = torch.zeros(S, M, H, dtype=torch.float64, device="cuda")
    e_car = torch.zeros_like(car)
    car[:S - 1] = lr.carried(dGa[1:], w_hh)
    e_car[:S - 1] = ACC * (dGa[1:].abs() @ w_hh.abs())
    dh_in = dhs.transpose(0, 1)[ts].double() if dhs is not None else torch.zeros_like(car)
    dc = torch.zeros(M, H, dtype=torch.float64, device="cuda")
    e_dc = torch.zeros_like(dc)
    gates, c = v["gates"].double(), v["c"].double()
    for p in range(S - 1, -1, -1):
        i, f, g, o = gates[p].chunk(4, -1)
        dh, dct, ref, dcp = lr.cell_backward(dh_in[p], car[p], dc, i, f, g, o, c[p + 1], c[p])
        e_dh = e_car[p] + 2.0 ** -24 * dh.abs()
        bnd, e_dct = cell_backward_bounds(e_dc, e_dh, dc, dh, dct, i, f, g, o, torch.tanh(c[p + 1]), c[p], ref)
        ck.bound("dG", dG[p], ref, bnd)
        dc, e_dc = dcp, e_dct * f.abs() + 2.0 ** -24 * dcp.abs()
    ck.gemm("dh", v["dh"], lr.carried(dGa[0], w_hh), dGa[0].abs() @ w_hh.abs())
    ck.bound("dc", v["dc"], dc, e_dc + 1e-38)
    if d.dh0 is not None:
        ck.exact("dh0", d.dh0, v["dh"])
        ck.exact("dc0", d.dc0, v["dc"])
    # hoisted: over the (p, m) rows of the stored per-step values
    DG = dGa.reshape(S * M, 4 * H)
    HP = (v["h_bf"] if d.bf else v["h"])[:S].double().reshape(S * M, H)
    XT = v["xt"].double().reshape(S * M, d.I)
    ref = lr.hoisted_gradients(DG, HP, XT, w_ih)
    ck.gemm("g_w_hh", d.grads["g_w_hh"], ref["g_w_hh"], DG.abs().t() @ HP.abs())
    ck.gemm("g_w_ih", d.grads["g_w_ih"], ref["g_w_ih"], DG.abs().t() @ XT.abs())
    D32 = dG.double().reshape(S * M, 4 * H)                                  # the bias sum reads the fp32 dG
    ck.gemm("g_b", d.grads["g_b_ih"], D32.sum(0), D32.abs().sum(0))
    ck.exact("g_b_hh", d.grads["g_b_hh"], d.grads["g_b_ih"])
    ck.gemm("dxt", v["dxt"].reshape(S * M, d.I), ref["dxt"], DG.abs() @ w_ih.abs())
    if dx is not None:
        want = lr.scatter(v["dxt"], d.reverse)                               # fp32: a permutation
        ck.exact("dx", dx, want if base is None else base + want)             # one fp32 addition
    if dhs is None and d.h0 is None:
        for k, t in list(d.grads.items()) + [("dh", v["dh"]), ("dc", v["dc"])] + ([("dx", dx)] if dx is not None else []):
            ck.value("%s without d hs" % k, t, 0.0)


def _run(case, seed, check=True):
    """Runs the case from sentinel-filled buffers, checking each call when ``check``; returns every output tensor."""
    precision, impl, layout, S, M, I, H, opts = _CASES[case]
    g = torch.Generator(device="cuda").manual_seed(seed)
    ck = Checker(case)
    if layout == "row":
        Hh, Ww = _row_shape()
        N, C, S, M = M, I, Ww, M * Hh
        dirs = [_Dir(precision, impl, S, M, I, H, rev, False, g) for rev in (False, True)]
        dt = dirs[0].dt
        feat = torch.randn(N, Hh, Ww, C, device="cuda", generator=g).to(dt)
        out = torch.full((N, Hh, Ww, 2 * H), SENTINEL, dtype=dt, device="cuda")
        dout = torch.randn(N, Hh, Ww, 2 * H, device="cuda", generator=g)
        dfeat = torch.full((N, Hh, Ww, C), SENTINEL, device="cuda")
        es = out.element_size()
        xv = _strided(feat.view(-1), 0, M, S, C, Ww * C, C)
        for dr in dirs:
            dr.fill()
        for k, dr in enumerate(dirs):
            a = dr.a
            a.x, a.x_row, a.x_step = feat.data_ptr(), Ww * C, C
            a.hs, a.hs_st = None, out.data_ptr() + k * H * es
            a.hs_row, a.hs_step = Ww * 2 * H, 2 * H
            a.dhs = dout.data_ptr() + k * H * 4
            a.dx, a.dx_row, a.dx_step, a.dx_accumulate = dfeat.data_ptr(), Ww * C, C, k
            dr.forward()
            if check:
                torch.cuda.synchronize()
                check_forward(ck, dr, xv, hs_st=_strided(out.view(-1), k * H, M, S, H, Ww * 2 * H, 2 * H))
                if k == 0:
                    ck.value("second direction's half of the output", out[..., H:], SENTINEL)
        for k, dr in enumerate(dirs):
            base = dfeat.clone() if k == 1 else None
            dr.backward()
            if check:
                torch.cuda.synchronize()
                check_backward(ck, dr, _strided(dout.view(-1), k * H, M, S, H, Ww * 2 * H, 2 * H),
                               _strided(dfeat.view(-1), 0, M, S, C, Ww * C, C),
                               None if base is None else _strided(base.view(-1), 0, M, S, C, Ww * C, C))
        outs = [out.clone(), dfeat.clone()] + [t for dr in dirs for t in dr.outputs()]
        return ck, outs
    dr = _Dir(precision, impl, S, M, I, H, "reverse" in opts, "h0" in opts, g)
    dr.fill()
    x = torch.randn(M, S, I, device="cuda", generator=g).to(dr.dt)
    hs = torch.full((M, S, H), SENTINEL, device="cuda")
    dhs = None if "nograd" in opts else torch.randn(M, S, H, device="cuda", generator=g)
    a = dr.a
    a.x, a.x_row, a.x_step = x.data_ptr(), S * I, I
    a.hs, a.hs_row, a.hs_step = hs.data_ptr(), S * H, H
    hs_st = None
    if layout == "plain":
        hs_st = torch.full((M, S, H), SENTINEL, dtype=dr.dt, device="cuda")
        a.hs_st = hs_st.data_ptr()
    dr.forward()
    if check:
        torch.cuda.synchronize()
        check_forward(ck, dr, x, hs=hs, hs_st=hs_st)
    if layout == "l2":
        dx = dhs                                                            # DecoderLayer2.backward_inplace: d x over d hs
        dhs_before = dhs.clone()
    else:
        dx = torch.full((M, S, I), SENTINEL, device="cuda")
        dhs_before = dhs
    a.dhs = dhs.data_ptr() if dhs is not None else None
    a.dx, a.dx_row, a.dx_step, a.dx_accumulate = dx.data_ptr(), S * I, I, 0
    dr.backward()
    if check:
        torch.cuda.synchronize()
        check_backward(ck, dr, dhs_before, dx)
    return ck, [hs.clone(), dx.clone()] + ([hs_st.clone()] if hs_st is not None else []) + dr.outputs()


@pytest.mark.parametrize("schedule,case", _PARAMS, ids=["%s-%s" % sc for sc in _PARAMS])
def test_lstm_seq_steps_vs_float64(schedule, case):
    """Every stored per-step quantity of the forward and backward, the hoisted gradients and d x within the bounds of the
    module docstring of float64 from the kernels' own operands.  Under "deterministic" two runs must agree bit for bit."""
    from latex_ocr_b200 import _lib
    opts, _ = _SCHEDULES[schedule]
    seed = sorted(_CASES).index(case)
    with _lib.option(**opts):
        ck, first = _run(case, seed)
        if "deterministic" in opts:
            _, again = _run(case, seed, check=False)
            torch.cuda.synchronize()
            for a, b in zip(first, again):
                assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "deterministic: two runs differ"
    for k, v in ck.worst.items():
        _WORST[k] = max(_WORST.get(k, 0.0), v)
    print("\n%-24s %s" % ("%s %s" % (schedule, case), "  ".join("%s %.3f" % kv for kv in sorted(ck.worst.items()))))


def test_zz_worst_ratios():
    """Prints the worst |y - ref| / bound per quantity over the cases above (run after them)."""
    if not _WORST:
        pytest.skip("run with the step tests")
    print("\nworst |y - ref| / bound per quantity:")
    for k, v in sorted(_WORST.items()):
        print("  %-28s %.4f" % (k, v))
