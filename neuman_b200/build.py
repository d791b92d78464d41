"""Builds libneuman_b200.so (the C-ABI library) in-tree with nvcc for sm_90a (H100).

    python -m neuman_b200.build [--force]

Per-file flags: the stage kernels that mirror chains of separately-rounded torch ops are compiled
with -fmad=false; the MLP kernels keep FMA contraction.  No --use_fast_math anywhere (sin/cos of the
positional encoding must be the accurate versions).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libneuman_b200.so")
OBJ = os.path.join(HERE, "build")

SOURCES = {           # file -> extra flags
    "api.cu": [],
    "rays.cu": ["-fmad=false"],
    "composite.cu": ["-fmad=false"],
    "resample.cu": ["-fmad=false"],
    "render.cu": ["-fmad=false"],
    "warp.cu": [],
    "smpl.cu": [],
    "human_train.cu": [],
    "mlp_simt.cu": [],
    "mlp_tc.cu": [],
    "mlp_tc_bwd.cu": [],
    "dw_gemm.cu": [],
}
COMMON = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
          "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include"), "-I", CSRC]


def nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(ROOT, "include", "neuman_b200.h"))
    objs = []
    procs = []
    for src, extra in SOURCES.items():
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + headers):
            cmd = [nvcc()] + COMMON + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc failed on {src} ---\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(f"--- {src} ---\n{out}\n")
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or _stale(OUT, objs):
        cmd = [nvcc(), "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
        subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
