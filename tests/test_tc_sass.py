"""What ptxas makes of the tensor-core kernels (compiled here for sm_90a with the library's own flags; no GPU needed):
no wgmma serialised by the compiler (warning C7520), no register spills, and in the forward kernel's SASS a wait for
wgmma completion only at k-block and step boundaries, not after every HGMMA."""
import os
import re
import shutil
import subprocess

import pytest

from neuman_b200 import build as B

FILES = ("mlp_tc.cu", "mlp_tc_bwd.cu", "dw_gemm.cu")
FWD = ("_Z8k_mlp_tcILb0EEv8TcParams", "_Z8k_mlp_tcILb1EEv8TcParams")     # k_mlp_tc<false> (render), <true> (training)


def _nvcc():
    try:
        c = B.nvcc()
    except RuntimeError:
        return None
    return c if os.path.isabs(c) or shutil.which(c) else None


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("tc_sass")
    procs = {}
    for f in FILES:
        cmd = [nvcc] + B.COMMON + B.SOURCES[f] + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, f),
                                                  "-o", str(out / f.replace(".cu", ".o"))]
        procs[f] = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    logs = {}
    for f, p in procs.items():
        logs[f] = p.communicate()[0]
        assert p.returncode == 0, logs[f]
    return out, logs


def _functions(log):
    """entry function -> (stack bytes, spill store bytes, spill load bytes) from ptxas -v"""
    res = {}
    for m in re.finditer(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*Function properties[^\n]*\n\s*(\d+) bytes stack "
                         r"frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log):
        res[m.group(1)] = tuple(int(m.group(i)) for i in (2, 3, 4))
    return res


@pytest.mark.parametrize("f", FILES)
def test_no_serialised_wgmma(compiled, f):
    _, logs = compiled
    assert "C7520" not in logs[f], [ln for ln in logs[f].splitlines() if "C7520" in ln]


@pytest.mark.parametrize("f", FILES)
def test_tensor_core_kernels_do_not_spill(compiled, f):
    fns = _functions(compiled[1][f])
    kernels = {k: v for k, v in fns.items() if re.search(r"k_mlp_tc|k_dw_gemm", k)}
    assert kernels, fns
    for k, (_, st, ld) in kernels.items():
        assert st == 0 and ld == 0, (k, st, ld)


def test_forward_stack_frames(compiled):
    fns = _functions(compiled[1]["mlp_tc.cu"])
    assert fns[FWD[0]][0] == 0, fns[FWD[0]]
    assert fns[FWD[1]][0] <= 64, fns[FWD[1]]


@pytest.mark.parametrize("fn", FWD)
def test_forward_waits_only_at_group_boundaries(compiled, fn):
    out, _ = compiled
    cuobjdump = os.path.join(os.path.dirname(_nvcc()), "cuobjdump") if os.path.isabs(_nvcc()) else shutil.which("cuobjdump")
    if not cuobjdump or not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([cuobjdump, "-sass", "-fun", fn, str(out / "mlp_tc.o")], capture_output=True, text=True,
                          check=True).stdout
    n_mma = len(re.findall(r"\bHGMMA\.64x(?:256|128|16)x16\.F32\b", sass))
    n_wait0 = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", sass))
    n_wait1 = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", sass))
    assert n_mma >= 3, sass[:2000]
    # one wait<1> per k-block commit and one wait<0> per step in the source; a serialised kernel waits after each HGMMA
    assert n_wait1 >= 1 and n_wait0 < n_mma / 2, (n_mma, n_wait0, n_wait1)
