"""NeRF-T nets (the reference's --ablate_nerft background nets: position input (x, y, z, t)) without a GPU: the oracle's
stages against the reference's outputs (tests/golden/nerft.npz, tools/make_golden_nerft.py), which Joiners the drop-in
sends to the library, the CPU fall-through, and what ptxas makes of the NeRF-T forward kernel."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import neuman_b200 as nb
from neuman_b200 import autograd
from neuman_b200 import build as B
from neuman_b200.dropin import supported_joiner
from oracle import neuman_oracle as no
from tests import nerft_cases as nc
from tests import util

NERFT_FWD = ("_Z14k_mlp_tc_nerftILb0EEv8TcParams", "_Z14k_mlp_tc_nerftILb1EEv8TcParams")   # render, training forward


def nerft(**over):
    c, _ = nb.build_nerf(nb.default_opt(use_cuda=False, raw_pos_dim=4, **over))
    return c


@pytest.fixture(scope="module")
def gold():
    return util.golden("nerft.npz")


# ---- host logic ----------------------------------------------------------------------------------
def test_supported_joiner_accepts_posenc_nerft_nets():
    j = nerft()
    assert j.pos_pe.input_dims == 4 and tuple(j.nerf.pts_linears[0].weight.shape) == (256, 84)
    assert tuple(j.nerf.pts_linears[5].weight.shape) == (256, 340)
    assert supported_joiner(j) and nb.ops.is_nerft(j) and not nb.ops.is_nerft(nb.build_nerf(nb.default_opt(use_cuda=False))[0])


def test_supported_joiner_rejects_rotate_and_view_independent_nerft_nets():
    assert not supported_joiner(nerft(posenc="rotate"))          # the reference's rotate mapping asserts a 3-D input
    assert not supported_joiner(nerft(use_viewdirs=False))       # view-independent NeRF-T: not built
    j = nerft()
    j.pos_pe.N_freqs = 8
    assert not supported_joiner(j)


def test_net_slot_refuses_unbuilt_nerft_kinds():
    for j in (nerft(posenc="rotate"), nerft(use_viewdirs=False)):
        with pytest.raises(NotImplementedError):
            nb.ops.net_slot(j, ctx=object())                     # refused before any library call


def test_nerft_input_gradients_are_refused():
    """Nothing in the reference differentiates through a NeRF-T net's inputs: the autograd path refuses to."""
    with pytest.raises(NotImplementedError):
        autograd.joiner_forward(nerft(), torch.zeros(4, 4, requires_grad=True), torch.zeros(4, 3))
    with pytest.raises(NotImplementedError):
        autograd.joiner_forward(nerft(), torch.zeros(4, 4), torch.zeros(4, 3, requires_grad=True))


# ---- the oracle against the reference (goldens) ---------------------------------------------------
def test_package_nets_equal_the_reference_nets(gold):
    """nb.build_nerf seeds the same NeRF-T weights as the reference: the oracle on them gives the reference's raw."""
    c, f = nc.nerft_nets(nb.build_nerf, nb.default_opt)
    pts, views = torch.from_numpy(gold["pts"]), torch.from_numpy(gold["views"])
    for name, j in (("coarse", c), ("fine", f)):
        with torch.no_grad():
            raw = no.net_forward(util.oracle_params(j), pts, views).numpy()
        assert np.abs(raw - gold[f"net_{name}"]).max() < 2e-5, name


def test_time_changes_the_output(gold):
    """The same 50 points at two times: the reference's raw differs, so the time column is a real input."""
    a, b = gold["net_coarse"][300:350], gold["net_coarse"][350:400]
    assert np.array_equal(gold["pts"][300:350, :3], gold["pts"][350:400, :3])
    assert np.abs(a - b).max() > 1e-2


@pytest.mark.parametrize("i", [0, 1])
def test_oracle_render_equals_reference(gold, i):
    f = util.golden("frames.npz")
    c, fn = nc.nerft_nets(nb.build_nerf, nb.default_opt)
    H, W = nc.VAN["H"], nc.VAN["W"]
    rgb, dep = nc.oracle_render(util.oracle_params(c), util.oracle_params(fn), f["van_K"], f["van_c2w"], H, W,
                                nc.frame_time(*nc.FRAMES[i]))
    assert np.abs(rgb - gold[f"van{i}_rgb"].reshape(-1, 3)).max() < 1e-5
    assert np.abs(dep - gold[f"van{i}_depth"].reshape(-1)).max() < 1e-4
    # the two frames render differently
    assert np.abs(gold["van0_rgb"] - gold["van1_rgb"]).max() > 5e-4


def test_dropin_falls_through_for_cpu_nerft_nets(gold):
    """Under install(), Joiner.forward of a NeRF-T net on CPU tensors runs the reference's own forward."""
    from tests.standin_reference import standin
    with standin() as r:
        nb.install()
        try:
            c, _ = nc.nerft_nets(r.vanilla.build_nerf, nb.default_opt)
            assert type(c).__module__ == "models.vanilla" and supported_joiner(c)
            with torch.no_grad():
                raw = c(torch.from_numpy(gold["pts"]), torch.from_numpy(gold["views"])).numpy()
            assert np.abs(raw - gold["net_coarse"]).max() < 2e-5
        finally:
            nb.dropin.uninstall()


# ---- the exact-window model of the time k-block ----------------------------------------------------
def test_window_model_of_the_time_slab_rejects_planted_defects(gold):
    """The windows of tests/tc_exact.py over the kernel's K order (nerft_cases.nerft_blocks) hold an fp16-operand layer-0
    output computed in that order, and reject the same output with the time slab dropped or with two time columns
    swapped (sin / cos of one frequency: a column-permutation slip in the packer)."""
    from tests import tc_exact as tx
    c, _ = nc.nerft_nets(nb.build_nerf, nb.default_opt)
    W16, _ = tx.weights(c, "cpu")
    pts = torch.from_numpy(gold["pts"]).double()
    with torch.no_grad():
        enc = no.embed(torch.from_numpy(gold["pts"]), util.oracle_params(c).pos_pe).double()
    pe96 = torch.cat([enc, torch.ones(pts.shape[0], 1, dtype=torch.float64), torch.zeros(pts.shape[0], 11, dtype=torch.float64)], 1)
    pe96 = tx.r16(pe96)
    e, B = tx.mma_ref(nc.nerft_blocks(W16, 0, pe96, None))

    def kernel(**defect):                   # an fp16 layer-0 output computed in the kernel's K order, maybe with a defect
        return tx.r16(tx.mma_ref(nc.nerft_blocks(W16, 0, pe96, None, **defect))[0].clamp_min(0.0))
    assert tx.check16("layer0", kernel(), e, B, relu=True).n_bad == 0
    assert tx.check16("layer0", kernel(time_slab=False), e, B, relu=True).n_bad > 0
    slip = nc.kernel_time_columns()
    slip[1], slip[2] = slip[2], slip[1]
    assert tx.check16("layer0", kernel(time_cols=slip), e, B, relu=True).n_bad > 0


# ---- what ptxas makes of the NeRF-T forward kernel --------------------------------------------------
@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    try:
        nvcc = B.nvcc()
    except RuntimeError:
        nvcc = None
    if nvcc is None or not (os.path.isabs(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("nerft_sass")
    cmd = [nvcc] + B.COMMON + B.SOURCES["mlp_tc.cu"] + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, "mlp_tc.cu"),
                                                       "-o", str(out / "mlp_tc.o")]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout
    return out / "mlp_tc.o", p.stdout


@pytest.mark.parametrize("fn,max_stack", [(NERFT_FWD[0], 0), (NERFT_FWD[1], 64)])
def test_nerft_kernel_neither_serialises_wgmma_nor_spills(ptxas_log, fn, max_stack):
    """No C7520 in the file, no spills; the render kernel has no stack frame, the training forward at most the 64 B of
    k_mlp_tc<true> (its lane-indexed sign words)."""
    _, log = ptxas_log
    assert "C7520" not in log, [ln for ln in log.splitlines() if "C7520" in ln]
    m = re.search(r"Compiling entry function '%s'[^\n]*\n[^\n]*Function properties[^\n]*\n\s*(\d+) bytes stack "
                  r"frame, (\d+) bytes spill stores, (\d+) bytes spill loads" % fn, log)
    assert m, fn + " not compiled"
    stack, st, ld = (int(m.group(i)) for i in (1, 2, 3))
    assert stack <= max_stack and st == 0 and ld == 0, (fn, stack, st, ld)


@pytest.mark.parametrize("fn", NERFT_FWD)
def test_nerft_kernel_waits_only_at_group_boundaries(ptxas_log, fn):
    """In the SASS of k_mlp_tc_nerft the waits for wgmma completion are one wait<1> per k-block commit and one wait<0>
    per step, as in the source: a serialised kernel would wait after every HGMMA (the rule of tests/test_tc_sass.py)."""
    obj, _ = ptxas_log
    nvcc = B.nvcc()
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump") if os.path.isabs(nvcc) else shutil.which("cuobjdump")
    if not cuobjdump or not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([cuobjdump, "-sass", "-fun", fn, str(obj)], capture_output=True, text=True,
                          check=True).stdout
    n_mma = len(re.findall(r"\bHGMMA\.64x(?:256|128|16)x16\.F32\b", sass))
    n_wait0 = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", sass))
    n_wait1 = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", sass))
    assert n_mma >= 3, sass[:2000]
    assert n_wait1 >= 1 and n_wait0 < n_mma / 2, (n_mma, n_wait0, n_wait1)
