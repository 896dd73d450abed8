"""(build the timing variant first: LO_LIB_DIR=_C_timing LO_NVCC_EXTRA=-DLO_ATT_TIMING python -m latex_ocr_b200.build)
Per-CTA timeline of the attention step kernels (timing build: LO_LIB_DIR=_C_timing, built with -DLO_ATT_TIMING).
Stamps (%globaltimer, ns): 0 entry, 1 consumer past griddepcontrol.wait, 2 consumer prologue done, 3 first stage landed,
4 main loop done, 8 after the CTA barrier, 9 last ticket taken (cluster-free combine), 5 exit; producer: 6 first stage issued,
7 last stage issued.  Both grids of the forward and the tensor-core backward are timed in one run: att_cluster=2 (every launch a
cluster) and att_cluster=1 (the default: cluster-free when that grid is one resident wave); per launch it reports the CTAs that
enter more than 5 us after the first one (a second wave), the launch span and the median main loop."""
import ctypes, os, sys
os.environ.setdefault("LO_LIB_DIR", "_C_timing")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import bench_support as bs
from latex_ocr_b200 import _lib
from latex_ocr_b200.img2seq import Img2SeqModel
from latex_ocr_b200.data import SimpleVocab

B, T = 64, 150
class Cfg:
    encoder_cnn = "vanilla"; positional_embeddings = True; lr_init = 1e-3; lr_method = "adam"; cuda_graph = False
m = Img2SeqModel(Cfg(), vocab=SimpleVocab(500), device="cuda:0", precision="bf16", impl="tc")
m.build_train(); m.train_mode(True)
img, formula = bs.synthetic_batch(B, 128, 512, 500, T, seed=1234)
img, formula = img.cuda(), formula.cuda()
for _ in range(2):
    m.train_step(img, formula)
torch.cuda.synchronize()
L = _lib.lib()
dec, enc = m.decoder, m.encoder
key = [k for k in dec._ws if k[0] == B and k[1] == T][0]
R = key[2]
ws = dec._ws[key]
t, a = ws["t"], ws["args"]
A = C = 512
O1 = A + C + 4 * 512
enc_out = enc._ws[(B, 128, 512)]["out"].view(B, R, C)
st = _lib.stream_ptr()
dt = _lib.LO_BF16
buf = torch.zeros(1024 * 16, dtype=torch.int64, device="cuda")
_lib.check(L.lo_debug_buffer(_lib.ptr(buf)))
_lib.set_option("att_abi_pdl", 1)       # static inputs: let the stand-alone entry points overlap like the time loop's launches do


def fwd(s):
    o1 = t["out1"][s]
    _lib.check(L.lo_attention_forward_mask(_lib.ptr(t["att1"]), _lib.ptr(enc_out), dt, _lib.ptr(o1), O1, a.w_full,
                                           ctypes.c_void_p(t["alphas"].data_ptr() + s * R * 4), T * R, _lib.ptr(t["ctx"][s]),
                                           None, 0, None, _lib.ptr(t["att_mask"][s]), B, R, A, C, _lib.ptr(t["work"]), st))


def bwd(s):
    o1 = t["out1"][s]
    _lib.check(L.lo_attention_backward(_lib.ptr(t["att1"]), _lib.ptr(enc_out), dt, _lib.ptr(o1), ctypes.c_void_p(o1.data_ptr() + A * 4), O1,
                                       a.w_full, ctypes.c_void_p(t["alphas"].data_ptr() + s * R * 4), T * R, _lib.ptr(t["ctx"][s]),
                                       _lib.ptr(t["dxh"]), C + 512, _lib.ptr(t["dreg"]), R, ctypes.c_void_p(t["sreg"].data_ptr() + s * 4), T,
                                       ctypes.c_void_p(t["de"].data_ptr() + s * R * 4), _lib.ptr(t["dcat"][s]),
                                       ctypes.c_void_p(t["dcat"][s].data_ptr() + A * 4), O1, _lib.ptr(t["dctx"][s]), None,
                                       _lib.ptr(t["att_mask"][s]), B, R, A, C, _lib.ptr(t["work"]), st))


def report(name, n=256):
    x = buf.cpu().numpy().reshape(-1, 16)[:n].astype(np.float64)
    t0 = x[:, 0].min()
    late = int(((x[:, 0] - t0) > 5e3).sum())
    wave2 = int((x[:, 0] > x[:, 5].min()).sum())        # entered only after a CTA of the same launch had exited
    loop = np.median(x[:, 4] - x[:, 3]) / 1e3
    span = (x[:, 5].max() - t0) / 1e3
    def col(k):
        v = (x[:, k] - t0) / 1e3
        return "%6.2f / %6.2f / %6.2f" % (v.min(), np.median(v), v.max())
    print("== %s (us after the first CTA's entry; min / median / max over %d CTAs)" % (name, n))
    for k, lab in ((0, "entry"), (6, "producer: first stage issued"), (1, "consumer past griddepcontrol.wait"), (2, "consumer prologue done"),
                   (3, "first stage landed"), (7, "producer: last stage issued"), (4, "main loop done"), (8, "after CTA barrier"), (5, "exit")):
        print("  %-36s %s" % (lab, col(k)))
    print("  span first entry -> last exit: %.2f us" % span, flush=True)
    print("  summary: %d of %d CTAs enter > 5 us after the first (under PDL the first ones enter during the preceding launch), "
          "%d after a CTA of this launch exited (second wave), span %.2f us, median main loop (first stage -> loop done) %.2f us" % (
              late, n, wave2, span, loop), flush=True)


for cl in (2, 1):
    _lib.set_option("att_cluster", cl)
    for name, fn in (("forward (mask emission), back-to-back launches", fwd), ("backward (mma), back-to-back launches", bwd)):
        name = "%s, att_cluster=%d" % (name, cl)
        for rep in range(2):
            buf.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for s in range(40):
                fn(s)
            e1.record(); torch.cuda.synchronize()
        print("%s: %.2f us per launch" % (name, e0.elapsed_time(e1) / 40 * 1e3))
        report(name)
_lib.set_option("att_cluster", 1)
# in situ: one eager train step; the last attention launch is the backward of step 0
m.train_step(img, formula); torch.cuda.synchronize()
report("backward of step 0 inside a train step (eager launches)")
_lib.check(L.lo_debug_buffer(None))
