"""Where the weight-gradient time goes: every tc_wgrad_kernel launch of the cfg #2 train step (B = 64, 128 x 512 images,
T = 150, bf16), timed at the step's own shapes.

  python tools/wgrad_waves.py [--iters 100] [--json OUT]

Per launch: the time of one library call from CUDA events over --iters calls (the call also clears its fp32 output), the
kernel's own time, grid and shared memory from a torch.profiler trace taken in a separate pass, the FLOPs from the shapes,
TFLOP/s of the kernel and the number of waves (grid over resident CTAs: one CTA per SM at the kernel's shared memory).
The "2-wave probe" rows run datt1^T enc with a smaller batch, which gives a grid of at most two waves: the in-wave rate.
The card's name, power limit and max SM clock are read in the same call.  LO_LIB_DIR selects the library build.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from latex_ocr_b200 import _lib  # noqa: E402

B, T, R = 64, 150, 14 * 62
SM_SMEM = 228 * 1024          # H100 shared memory per SM; each resident block also reserves 1 KB

# (name, Cin, Cout, H, W, pad) of conv2..conv6 at 128 x 512 input images
CONVS = [("conv2 wgrad", 64, 128, 64, 256, 1), ("conv3 wgrad", 128, 256, 32, 128, 1), ("conv4 wgrad", 256, 256, 32, 128, 1),
         ("conv5 wgrad", 256, 512, 16, 128, 1), ("conv6 wgrad", 512, 512, 16, 64, 0)]
# (name, M, N, K) of the decoder backward's hoisted C[M][N] = A[K][M]^T B[K][N]
GEMMS = [("dcat^T h", 3072, 512, B * T), ("dG^T gctx", 2048, 512, B * T), ("onehot^T dG", 504, 2048, B * T),
         ("datt1^T enc", 512, 512, B * R), ("datt1^T enc, B=16 (2-wave probe)", 512, 512, 16 * R)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = "nvidia-smi unavailable (%s)" % e
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q, "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def launches():
    L = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(0)
    out = []
    for name, cin, cout, h, w, pad in CONVS:
        ho, wo = h + 2 * pad - 2, w + 2 * pad - 2
        x = torch.randn(B, h, w, cin, device="cuda", generator=g).bfloat16()
        dy = torch.randn(B, ho, wo, cout, device="cuda", generator=g).bfloat16()
        dw = torch.empty(cout, 3, 3, cin, device="cuda")

        def call(x=x, dy=dy, dw=dw, h=h, w=w, cin=cin, cout=cout, pad=pad):
            _lib.check(L.lo_conv3x3_wgrad(_lib.ptr(x), _lib.ptr(dy), _lib.ptr(dw), None, _lib.LO_BF16, B, h, w, cin, cout, pad,
                                          _lib.LO_IMPL_TC, _lib.stream_ptr()))
        out.append((name, 2.0 * B * ho * wo * 9 * cin * cout, call))
    for name, m, n, k in GEMMS:
        a = torch.randn(k, m, device="cuda", generator=g).bfloat16()
        b = torch.randn(k, n, device="cuda", generator=g).bfloat16()
        c = torch.empty(m, n, device="cuda")

        def call(a=a, b=b, c=c, m=m, n=n, k=k):
            # A[K][M], B[K][N] row-major with a clear fp32 C: lo_gemm's tensor-core route to the TN weight-gradient kernel
            _lib.check(L.lo_gemm(_lib.ptr(a), _lib.LO_BF16, _lib.ptr(b), _lib.LO_BF16, _lib.ptr(c), _lib.LO_F32, m, n, k, 1, m, n, 1, n,
                                 1, 0, 0, 0, None, 0, 0, _lib.LO_IMPL_TC, _lib.stream_ptr()))
        out.append((name, 2.0 * m * n * k, call))
    return out


def event_ms(call, iters):
    for _ in range(5):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def traced(runs, reps, tmp):
    """{launch name: (kernel name, grid, dynamic + static shared memory, mean kernel us)} from one profiler pass."""
    from torch.profiler import ProfilerActivity, profile
    res = {}
    for name, _, call in runs:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call()
            torch.cuda.synchronize()
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel" and "tc_wgrad_kernel" in e.get("name", "")]
        if len(ev) != reps:
            raise RuntimeError("%s: expected %d tc_wgrad_kernel launches in the trace, found %d" % (name, reps, len(ev)))
        a = ev[-1]["args"]
        res[name] = (ev[-1]["name"], a["grid"], int(a.get("shared memory", 0)), sum(e["dur"] for e in ev) / reps)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--trace-reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("wgrad_waves: needs a CUDA device")
    info = card()
    runs = launches()
    times = {name: event_ms(call, args.iters) for name, _, call in runs}
    with tempfile.TemporaryDirectory() as tmp:
        tr = traced(runs, args.trace_reps, tmp)
    rows = []
    print("card: %s | %s | SMs %d | library %s" % (info["name"], info["nvidia_smi"], info["sms"], _lib.LIB_PATH))
    print("%-34s %-42s %-14s %6s %7s %10s %10s %8s" % ("launch", "kernel", "grid", "CTAs", "waves", "call us", "kernel us", "TFLOP/s"))
    for name, flop, _ in runs:
        kname, grid, smem, kus = tr[name]
        ctas = grid[0] * grid[1] * grid[2]
        per_sm = SM_SMEM // (smem + 1024)
        waves = ctas / (per_sm * info["sms"])
        short = kname.split("tc_wgrad_kernel")[1].split(">")[0] + ">"
        rows.append(dict(launch=name, kernel="tc_wgrad_kernel" + short, grid=grid, ctas=ctas, resident_per_sm=per_sm, waves=waves,
                         call_us=times[name] * 1e3, kernel_us=kus, gflop=flop / 1e9, tflops=flop / kus / 1e6))
        print("%-34s %-42s %-14s %6d %7.2f %10.1f %10.1f %8.0f" % (name, "tc_wgrad_kernel" + short, "x".join(map(str, grid)), ctas, waves,
                                                                   times[name] * 1e3, kus, flop / kus / 1e6))
    step = [r for r in rows if "probe" not in r["launch"]]
    print("sum over the step's launches: kernel %.1f us, call %.1f us, %.1f GFLOP" % (sum(r["kernel_us"] for r in step),
                                                                                  sum(r["call_us"] for r in step), sum(r["gflop"] for r in step)))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "library": _lib.LIB_PATH, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
