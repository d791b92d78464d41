"""TEST INFRASTRUCTURE ONLY -- builds (g++) and binds (ctypes) the host emulation of the human-trainer kernels: the same
kernel bodies as libneuman_b200.so compiles for sm_90a (neuman_b200/csrc/human_train_kernels.cuh,
smpl_train_kernels.cuh), executed serially on numpy arrays.  See cuda_emu.h."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "neuman_b200", "csrc")
OUT = os.path.join(HERE, "_build", "libhuman_train_emu.so")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    srcs = [os.path.join(HERE, "human_train_emu.cpp")]
    deps = srcs + [os.path.join(HERE, "cuda_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith("_kernels.cuh")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-I", CSRC, "-I", HERE]
                              + srcs + ["-o", OUT])
    _lib = C.CDLL(OUT)
    return _lib


def ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)
