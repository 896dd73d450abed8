import os, sys, ctypes
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from latex_ocr_b200 import _lib
L = _lib.lib()
dbg = torch.zeros(128, dtype=torch.int64, device="cuda")
N, H, W, Cin, Cout = 64, 32, 128, 256, 256
x = torch.randn(N, H, W, Cin, device="cuda").bfloat16(); w = (torch.randn(Cout, 3, 3, Cin, device="cuda") * 0.02).bfloat16()
b = torch.zeros(Cout, device="cuda"); y = torch.zeros(N, H, W, Cout, device="cuda", dtype=torch.bfloat16)
def run():
    _lib.check(L.lo_conv3x3(_lib.ptr(x), _lib.ptr(w), _lib.ptr(b), None, _lib.ptr(y), 1, N, H, W, Cin, Cout, 1, 1, 1, _lib.stream_ptr()))
for mc in (0, 1):
    _lib.set_option("conv_mc", mc)
    for _ in range(3): run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10): run()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    fl = 2.0 * N * H * W * Cout * Cin * 9
    L.lo_debug_buffer(ctypes.c_void_p(dbg.data_ptr())); run(); torch.cuda.synchronize(); L.lo_debug_buffer(None)
    d = dbg.cpu().tolist()
    print("conv 256->256 32x128 B=64 mc=%d: %.1f us  %.0f TFLOP/s" % (mc, ms * 1e3, fl / ms / 1e9))
    print("  setup %d  first-full %d  last-commit %d  tmem-full %d  epi-done %d  end %d" % (d[1]-d[0], d[4]-d[0], d[5]-d[0], d[6]-d[0], d[10]-d[0], d[8]-d[0]))
    print("  producer issue deltas:", [d[64+k+1]-d[64+k] for k in range(0, 36)])
    print("  mma full-arrival deltas:", [d[16+k+1]-d[16+k] for k in range(0, 35)])
