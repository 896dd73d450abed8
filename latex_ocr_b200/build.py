"""In-tree build of the C-ABI library: nvcc -> latex_ocr_b200/_C/liblatex_ocr_b200.so (sm_90a only)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, os.environ.get("LO_LIB_DIR", "_C"))      # LO_LIB_DIR: build a tuning variant next to the product library
LIB = os.path.join(OUT, "liblatex_ocr_b200.so")
SOURCES = ["lo_gemm.cu", "lo_conv.cu", "lo_decoder.cu", "lo_attention.cu", "lo_skinny.cu", "lo_cluster.cu", "lo_optim.cu", "lo_tc.cu", "lo_scst.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v"] + os.environ.get("LO_NVCC_EXTRA", "").split()


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.sep not in c or os.path.exists(c)):
            return c
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OUT, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "latex_ocr_b200.h"))
    jobs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OUT, s.replace(".cu", ".o"))
        if force or _stale(obj, [src] + headers):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [_nvcc()] + NVCC_FLAGS + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        with open(obj.replace(".o", ".log"), "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, r.stderr[-4000:]))
        return src

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for s in ex.map(compile_one, jobs):
                if verbose:
                    print("compiled", s)
    objs = [os.path.join(OUT, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(LIB, objs):
        cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stderr[-4000:])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
