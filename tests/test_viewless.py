"""View-independent nets (use_viewdirs=False) without a GPU: the oracle's use_viewdirs=False path against the reference's
outputs (tests/golden/viewless.npz, tools/make_golden_viewless.py), which Joiners the drop-in sends to the library, the CPU
fall-through, what ptxas makes of the new kernels, and the exact-window rule of the output head."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import neuman_b200 as nb
from neuman_b200 import build as B
from neuman_b200.dropin import supported_joiner
from oracle import neuman_oracle as no
from oracle import synth_smpl
from tests import util
from tests import viewless_cases as vc
from tests.viewless_cases import head_check

NOVIEW = ("_Z15k_mlp_tc_noviewILb0EEv8TcParams", "_Z15k_mlp_tc_noviewILb1EEv8TcParams")
NOVIEW_BWD = "_Z19k_mlp_tc_bwd_noview8BwParams"


def viewless(posenc="posenc", **over):
    c, _ = nb.build_nerf(nb.default_opt(use_cuda=False, use_viewdirs=False, posenc=posenc, **over))
    return c


# ---- host logic ----------------------------------------------------------------------------------
def test_supported_joiner_accepts_view_independent_nets():
    assert supported_joiner(viewless("posenc")) and supported_joiner(viewless("rotate"))
    j = viewless()
    j.dir_pe.N_freqs = 7                                        # the direction encoding is never used
    assert supported_joiner(j)


def test_supported_joiner_rejects_other_shapes():
    off = nb.models.build_offset_net(nb.default_opt(use_cuda=False, num_offset_nets=1))
    assert not supported_joiner(nb.Joiner(off.pos_pe, off.pos_pe, off.nerf))          # OffsetNet: output_linear [3,256]
    j = viewless()
    j.nerf.scale_type = "linear"
    assert not supported_joiner(j)
    assert not supported_joiner(viewless(nerf_depth=6))
    j = viewless()
    j.pos_pe.N_freqs = 8
    assert not supported_joiner(j)


def test_viewless_cpu_tensors_fail_loudly():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        viewless()(torch.zeros(4, 3))


# ---- the oracle's use_viewdirs=False path against the reference (goldens) ---------------------------
@pytest.fixture(scope="module")
def gold():
    return util.golden("viewless.npz")


@pytest.mark.parametrize("pe", ["posenc", "rotate"])
def test_oracle_nets_against_reference(gold, pe):
    s = util.golden("stages.npz")
    pts, views = torch.from_numpy(s["n_pts"]), torch.from_numpy(s["n_views"])
    for name, j in zip(("coarse", "fine"), vc.viewless_nets(nb.build_nerf, nb.default_opt, pe)):
        assert vc.checksum(j) == gold[f"net_{pe}_{name}_sum"], "product nets are not seeded like the reference's"
        with torch.no_grad():
            y = no.net_forward(util.oracle_params(j), pts, views)
        assert np.abs(y.numpy() - gold[f"net_{pe}_{name}"]).max() <= 1e-6, (pe, name)


def test_oracle_render_vanilla_against_reference(gold):
    f = util.golden("frames.npz")
    c, fn = vc.viewless_nets(nb.build_nerf, nb.default_opt, "posenc")
    H, W = vc.VAN["H"], vc.VAN["W"]
    rgb, dep = no.render_vanilla(util.oracle_params(c), util.oracle_params(fn), f["van_K"], f["van_c2w"], H, W, 0.0, 3.14,
                                 samples_per_ray=vc.VAN["S"], importance_samples_per_ray=vc.VAN["N"])
    assert np.allclose(rgb.reshape(H, W, 3), gold["van_rgb"], atol=2e-6)
    assert np.allclose(dep.reshape(H, W), gold["van_depth"], atol=2e-6)


def test_oracle_human_renders_against_reference(gold):
    f = util.golden("frames.npz")
    H, W, S, N = vc.HUM["H"], vc.HUM["W"], vc.HUM["S"], vc.HUM["N"]
    K, c2w = f["h_K"], f["h_c2w"]
    b1 = synth_smpl.random_body(seed=1, center=(0.1, 0.0, 0.3))
    b2 = synth_smpl.random_body(seed=4, center=(-0.15, 0.0, 0.5))
    geo = b1["geo_threshold"]
    models = {k: vc.human_model(nb.HumanNeRF, nb.default_opt, k) for k in vc.HUMANS}
    P = {}
    for k, m in models.items():
        parts = (m.coarse_bkg_net, m.fine_bkg_net, m.coarse_human_net)
        assert np.array_equal(np.array([vc.checksum(j) for j in parts]), gold[f"human{k}_sums"]), k
        P[k] = [util.oracle_params(j) for j in parts]
    for can in (1, 0):
        r, d, a = no.render_smpl_nerf(P["A"][2], K, c2w, H, W, b1["verts"], b1["faces"], b1["Ts"], samples_per_ray=S,
                                      render_can=bool(can), geo_threshold=geo)
        assert 0 < (gold[f"smpl{can}_acc"] > 0).sum() < H * W           # hits and misses
        assert np.allclose(r.reshape(H, W, 3), gold[f"smpl{can}_rgb"], atol=2e-6)
        assert np.allclose(d.reshape(H, W), gold[f"smpl{can}_depth"], atol=2e-6)
        assert np.allclose(a.reshape(H, W), gold[f"smpl{can}_acc"], atol=2e-6)
    for k in vc.HUMANS:
        r, d = no.render_hybrid_nerf(*P[k], K, c2w, H, W, 0.0, 3.14, b1["verts"], b1["faces"], b1["Ts"], samples_per_ray=S,
                                     importance_samples_per_ray=N, geo_threshold=geo)[:2]
        assert np.allclose(r.reshape(H, W, 3), gold[f"hyb{k}_rgb"], atol=2e-6), k
        assert np.allclose(d.reshape(H, W), gold[f"hyb{k}_depth"], atol=2e-6), k
    r, d = no.render_hybrid_nerf_multi_persons(P["A"][0], P["A"][1], [P["A"][2], P["B"][2]], K, c2w, H, W, 0.0, 3.14,
                                               [b1["verts"], b2["verts"]], [b1["faces"]] * 2, [b1["Ts"], b2["Ts"]],
                                               samples_per_ray=S, importance_samples_per_ray=N, geo_threshold=geo)[:2]
    assert np.allclose(r.reshape(H, W, 3), gold["multi_rgb"], atol=2e-6)
    assert np.allclose(d.reshape(H, W), gold["multi_depth"], atol=2e-6)


# ---- SASS -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    try:
        nvcc = B.nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    if not (os.path.isabs(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("viewless_sass")
    logs = {}
    for f in ("mlp_tc.cu", "mlp_tc_bwd.cu"):
        r = subprocess.run([nvcc] + B.COMMON + B.SOURCES[f] + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, f), "-o",
                                                               str(out / f.replace(".cu", ".o"))],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        logs[f] = r.stdout + r.stderr
    return out, nvcc, logs


def _props(log, fn):
    m = re.search(r"Compiling entry function '%s'[^\n]*\n[^\n]*Function properties[^\n]*\n\s*(\d+) bytes stack frame, "
                  r"(\d+) bytes spill stores, (\d+) bytes spill loads" % fn, log)
    assert m, fn
    return tuple(int(g) for g in m.groups())


def test_viewless_kernels_compile_clean(compiled):
    _, _, logs = compiled
    for f, log in logs.items():
        bad = [ln for ln in log.splitlines() if "C7520" in ln and "noview" in ln]
        assert not bad, bad
    for fn in NOVIEW:
        stack, st, ld = _props(logs["mlp_tc.cu"], fn)
        assert st == 0 and ld == 0 and stack <= 64, (fn, stack, st, ld)
    assert _props(logs["mlp_tc_bwd.cu"], NOVIEW_BWD)[1:] == (0, 0)


@pytest.mark.parametrize("fn", NOVIEW)
def test_viewless_forward_waits_only_at_group_boundaries(compiled, fn):
    out, nvcc, _ = compiled
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump") if os.path.isabs(nvcc) else shutil.which("cuobjdump")
    if not cuobjdump or not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([cuobjdump, "-sass", "-fun", fn, str(out / "mlp_tc.o")], capture_output=True, text=True,
                          check=True).stdout
    n_mma = len(re.findall(r"\bHGMMA\.64x(?:256|16)x16\.F32\b", sass))
    n_wait0 = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", sass))
    n_wait1 = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", sass))
    assert n_mma >= 2 and n_wait1 >= 1 and n_wait0 < n_mma / 2, (n_mma, n_wait0, n_wait1)


# ---- the exact-window rule of the output head (tests/viewless_cases.py head_check) ----------------
def _head_case(n=300, seed=0):
    g = torch.Generator().manual_seed(seed)
    x7 = torch.relu(torch.randn(n, 256, generator=g)).half()
    W = (torch.randn(4, 256, generator=g) * 0.06).float()
    b = (torch.randn(4, generator=g) * 0.3).float()
    sd = {'output_linear.weight': W, 'output_linear.bias': b}
    W16 = {k: v.half().double() for k, v in sd.items()}
    W32 = {k: v.double() for k, v in sd.items()}
    return x7, W, b, W16, W32


def _fp32_head(x7, W16w, bias, order):
    """fp32 evaluation of the head in a given summation order (what a correct kernel may produce)."""
    x, w = x7.float(), W16w.float()
    if order == "forward":
        acc = torch.zeros(x.shape[0], 4)
        for k0 in range(0, 256, 16):
            acc = acc + x[:, k0:k0 + 16] @ w[:, k0:k0 + 16].T
    else:
        acc = torch.zeros(x.shape[0], 4)
        for k in range(255, -1, -1):
            acc = acc + x[:, k:k + 1] * w[:, k][None]
    return acc + bias


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_head_window_accepts_fp32_evaluations(order):
    x7, W, b, W16, W32 = _head_case()
    raw = _fp32_head(x7, W16['output_linear.weight'], b, order)
    c = head_check(W16, W32, x7.double(), raw)
    assert c.n_bad == 0, c.message()


def test_head_window_rejects_defects():
    x7, W, b, W16, W32 = _head_case()
    w = W16['output_linear.weight']
    for name, raw in (("dropped bias", _fp32_head(x7, w, torch.zeros(4), "forward")),
                      ("fp16 bias", _fp32_head(x7, w, b.half().float(), "forward")),
                      ("swizzle slip", _fp32_head(x7[:, torch.arange(256) ^ 8], w, b, "forward"))):
        assert head_check(W16, W32, x7.double(), raw).n_bad > 0, name
