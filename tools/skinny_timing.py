import os, sys, ctypes
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from latex_ocr_b200 import _lib
L = _lib.lib()
dbg = torch.zeros(16, dtype=torch.int64, device="cuda")
for (M, N, K) in ((64, 3072, 512), (64, 2048, 512)):
    A = torch.randn(M, K, device="cuda").bfloat16(); W = torch.randn(N, K, device="cuda").bfloat16()
    C = torch.zeros(M, N, device="cuda"); b = torch.zeros(N, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    def run():
        _lib.check(L.lo_gemm(_lib.ptr(A), 1, _lib.ptr(W), 1, _lib.ptr(C), 0, M, N, K, K, 1, 1, K, N, 1, 0, 0, 0, _lib.ptr(b), 0, 0, 1, _lib.stream_ptr()))
    for cold in (0, 1):
        for it in range(3):
            run()
        L.lo_debug_buffer(ctypes.c_void_p(dbg.data_ptr()))
        if cold: flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record(); run(); e1.record(); torch.cuda.synchronize()
        L.lo_debug_buffer(None)
        d = dbg.cpu().tolist()
        names = ["start", "setup done", "1st TMA issued", "all TMA issued", "1st full", "last commit", "tmem full seen", "pre-dealloc", "end", "epi 1st tmem_ld done", "epi loop done"]
        print("M%d N%d K%d cold=%d  event %.1f us | cycles since start:" % (M, N, K, cold, e0.elapsed_time(e1) * 1e3), {n: d[i] - d[0] for i, n in enumerate(names)})
