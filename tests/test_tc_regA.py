"""The render instantiations of the forward MLP kernel (kTrain = false) keep each layer's output in registers as the next
layer's wgmma A operand: their hidden-layer HGMMAs take register A fragments, and between a step's last wgmma wait and the
next step's first HGMMA there is no shared-memory store (the epilogue packs into registers only).  Compiled here for
sm_90a with the library's own flags; no GPU needed."""
import os
import re
import shutil
import subprocess

import pytest

from neuman_b200 import build as B

RENDER = ("_Z8k_mlp_tcILb0EEv8TcParams", "_Z15k_mlp_tc_noviewILb0EEv8TcParams", "_Z14k_mlp_tc_nerftILb0EEv8TcParams")
HGMMA = re.compile(r"\bHGMMA\.64x(?:256|128|16)x16\.F32\b([^;]*);")


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    try:
        nvcc = B.nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)) and not shutil.which(nvcc):
        pytest.skip("nvcc not found")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump") if os.path.isabs(nvcc) else shutil.which("cuobjdump")
    if not cuobjdump or not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    obj = str(tmp_path_factory.mktemp("tc_rega") / "mlp_tc.o")
    subprocess.run([nvcc] + B.COMMON + B.SOURCES["mlp_tc.cu"] + ["-c", os.path.join(B.CSRC, "mlp_tc.cu"), "-o", obj],
                   check=True, capture_output=True)
    return {fn: subprocess.run([cuobjdump, "-sass", "-fun", fn, obj], capture_output=True, text=True, check=True).stdout
            for fn in RENDER}


def _a_operand(operands):
    """the A operand of an HGMMA: a general register (R..) or a descriptor (gdesc[UR..])"""
    m = re.match(r"\s*R\d+\s*,\s*(\S+)", operands)
    return m.group(1).rstrip(",")


@pytest.mark.parametrize("fn", RENDER)
def test_hidden_layers_take_register_a(sass, fn):
    ops = [_a_operand(m.group(1)) for m in HGMMA.finditer(sass[fn])]
    reg = [a for a in ops if re.fullmatch(r"R\d+", a)]
    desc = [a for a in ops if a.startswith("gdesc")]
    assert len(reg) + len(desc) == len(ops), ops[:8]
    # per tile: 4 K slices on each activation k-block (steps 1-9 / 1-8), the encoding and bias / time / direction
    # k-blocks from shared memory; the activation k-blocks are the majority
    assert len(reg) > 2 * len(desc) > 0, (len(reg), len(desc))


@pytest.mark.parametrize("fn", RENDER)
def test_no_shared_stores_between_steps(sass, fn):
    lines = sass[fn].splitlines()
    wait0 = [i for i, ln in enumerate(lines) if re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", ln)]
    mma = [i for i, ln in enumerate(lines) if HGMMA.search(ln)]
    assert len(wait0) >= 8, len(wait0)
    checked, tile_ends = 0, 0
    for w in wait0:
        nxt = [i for i in mma if i > w]
        if not nxt:
            continue
        gap = lines[w:nxt[0]]
        if any(re.search(r"\bBAR\.SYNC\b", ln) for ln in gap):
            tile_ends += 1          # the end of a tile: the next tile's encodings are stored behind the warpgroup barrier
            continue
        stores = [ln.strip() for ln in gap if re.search(r"\bSTS\b", ln)]
        assert not stores, (w, stores[:4])
        checked += 1
    assert tile_ends <= 1 and checked >= 7, (tile_ends, checked)
