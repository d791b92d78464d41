"""The drop-in on the GPU (SURVEY.md §8b): `neuman_b200.install()` rebinds the hot-path functions of modules with the
reference's names and signatures (tests/standin_reference.py: the reference tree itself is not needed), and the `render_*` /
sampler / `Joiner.forward` entry points are then called as `render_360.py`, `render_test_views.py`, `render_gathering.py`
and the trainers' validation call them -- with CUDA modules and tensors.  Results are compared with the goldens the
reference produced on the CPU."""
import contextlib
import io

import numpy as np
import pytest
import torch

import neuman_b200 as nb
from neuman_b200._lib import Context
from oracle import neuman_oracle as no
from oracle import scenes
from tests import util
from tests.standin_reference import standin

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope="module")
def ref():
    with standin() as r:
        r.mods = nb.install()
        assert nb.install()["render_utils"] is r.mods["render_utils"]       # idempotent
        yield r


def cap_of(ref, K, c2w, H, W, near=0.0, far=3.14):
    return nb.SimpleCapture(np.asarray(K), np.asarray(c2w).astype(np.float64), H, W, near, far)


def quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def launches():
    return Context.get(0).launch_count()


def test_reference_render_vanilla_runs_on_the_cuda_path(ref):
    f = util.golden("frames.npz")
    coarse, fine = scenes.seed_nets(ref.vanilla.build_nerf, nb.default_opt(use_cuda=True), 1)
    assert next(coarse.parameters()).is_cuda and type(coarse).__module__ == "models.vanilla"
    cap = cap_of(ref, f["van_K"], f["van_c2w"], 20, 28)
    l0 = launches()
    rgb, dep = quiet(ref.render_utils.render_vanilla, coarse, cap, fine_net=fine, rays_per_batch=100, samples_per_ray=48,
                     importance_samples_per_ray=40, return_depth=True)
    assert launches() > l0, "the reference's render_vanilla did not reach libneuman_b200"
    assert isinstance(rgb, np.ndarray) and rgb.dtype == np.float32 and rgb.shape == (20, 28, 3)
    cp, fp = no.net_params_from_joiner(coarse), no.net_params_from_joiner(fine)
    fl = util.floors16(lambda: no.render_vanilla(cp, fp, f["van_K"], f["van_c2w"], 20, 28, 0.0, 3.14, samples_per_ray=48,
                                                 importance_samples_per_ray=40))
    e_dep = np.abs(dep - f["van_depth"]).max()
    assert np.abs(rgb - f["van_rgb"]).max() < TOL and e_dep <= util.gate(e_dep, fl[1]), (e_dep, fl)
    cap = cap_of(ref, f["cfg1_K"], f["cfg1_c2w"], 64, 64)
    rgb, dep = quiet(ref.render_utils.render_vanilla, coarse, cap, fine_net=None, rays_per_batch=2048, samples_per_ray=64,
                     return_depth=True)
    assert np.abs(rgb - f["cfg1_rgb"]).max() < TOL and np.abs(dep - f["cfg1_depth"]).max() < TOL
    # a CPU model keeps the reference's own implementation (here its oracle restatement: the golden up to the host's BLAS
    # rounding)
    c_cpu, f_cpu = scenes.seed_nets(ref.vanilla.build_nerf, nb.default_opt(use_cuda=False), 1)
    l0 = launches()
    cap = cap_of(ref, f["van_K"], f["van_c2w"], 20, 28)
    rgb = quiet(ref.render_utils.render_vanilla, c_cpu, cap, fine_net=f_cpu, rays_per_batch=100, samples_per_ray=48,
                importance_samples_per_ray=40)
    assert launches() == l0 and np.abs(rgb - f["van_rgb"]).max() < 2e-6


def test_reference_human_renderers_run_on_the_cuda_path(ref):
    f = util.golden("frames.npz")
    torch.manual_seed(1)
    net = ref.human_nerf.HumanNeRF(nb.default_opt(num_offset_nets=0, use_cuda=False)).cuda()
    scenes.boost_density(net.coarse_human_net)
    sums = [scenes.net_checksum(net.coarse_bkg_net), scenes.net_checksum(net.fine_bkg_net), scenes.net_checksum(net.coarse_human_net)]
    assert np.allclose(sums, f["h_sum"], rtol=1e-6)
    b1, b2 = util.bodies()
    H, W = f["hyb_rgb"].shape[:2]
    cap = cap_of(ref, f["h_K"], f["h_c2w"], H, W)
    geo = b1["geo_threshold"]
    ru = ref.render_utils

    def close(a, gold, tol, what):
        bad = (np.abs(a - gold) > tol).reshape(H * W, -1).any(-1).mean()
        assert bad < 0.01, (what, bad, float(np.abs(a - gold).max()))      # grazing rays may flip hit/miss (see test_gpu_render.py)

    l0 = launches()
    for can in (1, 0):
        r, d, a = quiet(ru.render_smpl_nerf, net, cap, b1["verts"], b1["faces"], b1["Ts"], rays_per_batch=64, samples_per_ray=24,
                        render_can=bool(can), geo_threshold=geo, return_depth=True, return_mask=True, interval_comp=0.7)
        close(r, f[f"smpl{can}_rgb"], TOL, f"smpl{can} rgb")
        close(d, f[f"smpl{can}_depth"], TOL, f"smpl{can} depth")
        close(a, f[f"smpl{can}_acc"], TOL, f"smpl{can} acc")
    r, d = quiet(ru.render_hybrid_nerf, net, cap, b1["verts"], b1["faces"], b1["Ts"], rays_per_batch=64, samples_per_ray=24,
                 importance_samples_per_ray=16, geo_threshold=geo, return_depth=True)
    cb, fb, hp = (no.net_params_from_joiner(m) for m in (net.coarse_bkg_net, net.fine_bkg_net, net.coarse_human_net))
    fl_h = util.floors16(lambda: no.render_hybrid_nerf(cb, fb, hp, f["h_K"], f["h_c2w"], H, W, 0.0, 3.14, b1["verts"], b1["faces"],
                                                       b1["Ts"], samples_per_ray=24, importance_samples_per_ray=16,
                                                       geo_threshold=geo)[:2])
    close(r, f["hyb_rgb"], util.gate(0, fl_h[0]), "hybrid rgb")
    close(d, f["hyb_depth"], util.gate(0, fl_h[1]), "hybrid depth")
    r, d = quiet(ru.render_hybrid_nerf_multi_persons, net, cap, [net, net], [b1["verts"], b2["verts"]], [b1["faces"]] * 2,
                 [b1["Ts"], b2["Ts"]], rays_per_batch=64, samples_per_ray=24, importance_samples_per_ray=16, geo_threshold=geo,
                 return_depth=True)
    fl_m = util.floors16(lambda: no.render_hybrid_nerf_multi_persons(cb, fb, [hp, hp], f["h_K"], f["h_c2w"], H, W, 0.0, 3.14,
                                                                     [b1["verts"], b2["verts"]], [b1["faces"]] * 2,
                                                                     [b1["Ts"], b2["Ts"]], samples_per_ray=24,
                                                                     importance_samples_per_ray=16, geo_threshold=geo))
    close(r, f["multi_rgb"], util.gate(0, fl_m[0]), "multi rgb")
    close(d, f["multi_depth"], util.gate(0, fl_m[1]), "multi depth")
    assert launches() > l0


def test_reference_stage_functions_and_forward_on_cuda(ref):
    g = util.golden("stages.npz")
    ry, ru = ref.ray_utils, ref.render_utils
    dev = "cuda"
    with torch.no_grad():
        batch = {k: torch.from_numpy(g[n]).to(dev) for k, n in (("origin", "s_o"), ("direction", "s_d"), ("near", "s_near"), ("far", "s_far"))}
        l0 = launches()
        pts, dirs, z = ry.ray_to_samples(batch, 40, device=dev)
        assert launches() > l0
        assert np.abs(z.cpu().numpy() - g["s_z"]).max() < 2e-6 and np.abs(pts.cpu().numpy() - g["s_pts"]).max() < 2e-6
        raw = torch.from_numpy(g["c_raw"]).to(dev)
        outs = ru.raw2outputs(raw, z, batch["direction"], white_bkg=True)
        for name, t in zip(("rgb", "disp", "acc", "w", "depth"), outs):
            gold = g[f"c_{name}_1"]
            assert np.abs(t.cpu().numpy() - gold).max() <= 2e-5 * max(1.0, float(np.abs(gold).max())), name
        w = torch.from_numpy(g["c_w_1"]).to(dev)
        _, _, iz = ry.ray_to_importance_samples(batch, z, w, 24, device=dev)
        bad = (np.abs(iz.cpu().numpy() - g["i_z"]) > 2e-6).mean()
        assert bad < 0.01                                     # sample_pdf's `denom < 1e-5` discontinuity (see test_gpu_stages.py)
        coarse, _ = scenes.seed_nets(ref.vanilla.build_nerf, nb.default_opt(use_cuda=True), 1)
        l0 = launches()
        out = coarse(torch.from_numpy(g["n_pts"]).to(dev), torch.from_numpy(g["n_views"]).to(dev))
        assert launches() > l0 and np.abs(out.cpu().numpy() - g["n_coarse"]).max() < 1e-3
        # an architecture the kernels do not implement keeps the reference's own forward (install() never changes results)
        small, _ = scenes.seed_nets(ref.vanilla.build_nerf, nb.default_opt(use_cuda=True, nerf_width=128), 3)
        l0 = launches()
        x, v = torch.randn(50, 3, device=dev), torch.nn.functional.normalize(torch.randn(50, 3, device=dev), dim=-1)
        y = small(x, v)
        assert launches() == l0 and y.shape == (50, 4)
        nofreq, _ = scenes.seed_nets(ref.vanilla.build_nerf, nb.default_opt(use_cuda=True, pos_N_freqs=6, pos_max_freq=5), 3)
        assert nofreq(x, v).shape == (50, 4) and launches() == l0
    # under autograd (training) the reference's torch path runs unless install(train=True)
    out = coarse(torch.from_numpy(g["n_pts"]).to(dev), torch.from_numpy(g["n_views"]).to(dev))
    assert out.requires_grad
