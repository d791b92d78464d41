"""Pins the oracle (oracle/neuman_oracle.py) to the committed golden vectors, which were produced by
the unmodified reference (tools/make_golden.py).  Runs anywhere (no GPU, no reference tree)."""
import numpy as np
import pytest
import torch

from oracle import neuman_oracle as no
from tests import util

TOL = 2e-6


@pytest.fixture(autouse=True, scope="module")
def _one_thread():
    """CPU float32 reductions round differently with the number of threads they are split over: compare on one thread,
    so that the results do not depend on the host's core count"""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


def test_networks_have_reference_weights():
    g = util.golden("stages.npz")
    coarse, fine, human = util.product_nets()
    from oracle import scenes
    assert abs(scenes.net_checksum(coarse) - g["n_sum_coarse"]) < 1e-6 * g["n_sum_coarse"]
    assert abs(scenes.net_checksum(fine) - g["n_sum_fine"]) < 1e-6 * g["n_sum_fine"]
    assert abs(scenes.net_checksum(human) - g["n_sum_human"]) < 1e-6 * g["n_sum_human"]
    pts, views = torch.from_numpy(g["n_pts"]), torch.from_numpy(g["n_views"])
    with torch.no_grad():
        for net, key in ((coarse, "n_coarse"), (fine, "n_fine"), (human, "n_human")):
            y = no.net_forward(util.oracle_params(net), pts, views).numpy()
            assert np.abs(y - g[key]).max() < 5e-6


def test_rays_sampling_composite():
    g = util.golden("stages.npz")
    H, W = g["cam_HW"]
    o, d = no.shot_rays(g["cam_K"], g["cam_c2w"], no.all_pixel_coords(H, W))
    assert np.array_equal(o, g["rays_o0"]) and np.abs(d - g["rays_d0"]).max() < 1e-7
    o, d = no.shot_all_rays(g["cam_K"], g["cam_c2w"], H, W)
    assert np.abs(d.astype(np.float32) - g["rays_d1"]).max() < 1e-7
    so, sd = torch.from_numpy(g["s_o"]), torch.from_numpy(g["s_d"])
    near, far = torch.from_numpy(g["s_near"]), torch.from_numpy(g["s_far"])
    S = g["s_z"].shape[1]
    pts, _, z = no.ray_to_samples(so, sd, near, far, S)
    assert np.abs(z.numpy() - g["s_z"]).max() < TOL and np.abs(pts.numpy() - g["s_pts"]).max() < TOL
    _, _, zp = no.ray_to_samples(so, sd, near, far, S, perturb=1.0, t_rand=torch.from_numpy(g["s_trand"]))
    assert np.abs(zp.numpy() - g["s_z_perturb"]).max() < TOL
    _, _, zl = no.ray_to_samples(so, sd, near, far, S, lindisp=True)
    assert np.abs(zl.numpy() - g["s_z_lindisp"]).max() < TOL
    raw = torch.from_numpy(g["c_raw"])
    for wb in (1, 0):
        outs = no.raw2outputs(raw, torch.from_numpy(g["s_z"]), sd, white_bkg=bool(wb))
        for name, t in zip(("rgb", "disp", "acc", "w", "depth"), outs):
            ref = g[f"c_{name}_{wb}"]
            assert np.allclose(t.numpy(), ref, rtol=1e-5, atol=TOL), name
    w = torch.from_numpy(g["c_w_1"])
    N = g["i_z"].shape[1] - S
    pts, _, iz = no.ray_to_importance_samples(so, sd, torch.from_numpy(g["s_z"]), w, N)
    assert np.abs(iz.numpy() - g["i_z"]).max() < TOL and np.abs(pts.numpy() - g["i_pts"]).max() < 1e-5
    _, _, iz2 = no.ray_to_importance_samples(so, sd, torch.from_numpy(g["s_z"]), w, N, including_old=False)
    assert np.abs(iz2.numpy() - g["i_z_new"]).max() < TOL
    out = no.sample_pdf(torch.from_numpy(g["p_bins"]), torch.from_numpy(g["p_w"]), 11, det=False, u=torch.from_numpy(g["p_u"]))
    assert np.abs(out.numpy() - g["p_out"]).max() < TOL
    out = no.sample_pdf(torch.from_numpy(g["p_bins"]), torch.from_numpy(g["p_w"]), 11, det=True)
    assert np.abs(out.numpy() - g["p_out_det"]).max() < TOL


def test_near_far_and_warp():
    g = util.golden("stages.npz")
    from oracle import synth_smpl
    body = synth_smpl.random_body(seed=2, center=(0.1, 0.0, 0.3))
    n, f = no.geometry_guided_near_far(torch.from_numpy(g["nf_o"]), torch.from_numpy(g["nf_d"]),
                                       torch.from_numpy(body["verts"]), float(g["nf_thr"]))
    hit = ~np.isinf(g["nf_near"])
    assert np.array_equal(~torch.isinf(n).numpy(), hit) and hit.sum() > 0 and (~hit).sum() > 0
    assert np.abs(n.numpy()[hit] - g["nf_near"][hit]).max() < 2e-5 and np.abs(f.numpy()[hit] - g["nf_far"][hit]).max() < 2e-5
    cp, cd, cl = no.warp_samples_to_canonical(g["w_pts"], body["verts"], body["faces"], body["Ts"])
    assert np.abs(cp - g["w_can"]).max() < 1e-5 and np.abs(cd - g["w_dirs"]).max() < 1e-4
    assert np.abs(cl - g["w_closest"]).max() < 1e-5


def test_frames():
    f = util.golden("frames.npz")
    coarse, fine, _ = util.product_nets()
    cp, fp = util.oracle_params(coarse), util.oracle_params(fine)
    rgb, dep = no.render_vanilla(cp, None, f["cfg1_K"], f["cfg1_c2w"], 64, 64, 0.0, 3.14, rays_per_batch=2048,
                                 samples_per_ray=64)
    assert np.abs(rgb.reshape(64, 64, 3) - f["cfg1_rgb"]).max() < 5e-6
    assert np.abs(dep.reshape(64, 64) - f["cfg1_depth"]).max() < 5e-6
    rgb, dep = no.render_vanilla(cp, fp, f["van_K"], f["van_c2w"], 20, 28, 0.0, 3.14, samples_per_ray=48,
                                 importance_samples_per_ray=40)
    assert np.abs(rgb.reshape(20, 28, 3) - f["van_rgb"]).max() < 5e-6
    net = util.product_human_model()
    from oracle import scenes
    sums = [scenes.net_checksum(net.coarse_bkg_net), scenes.net_checksum(net.fine_bkg_net), scenes.net_checksum(net.coarse_human_net)]
    assert np.allclose(sums, f["h_sum"], rtol=1e-6)
    b1, b2 = util.bodies()
    hp = util.oracle_params(net.coarse_human_net)
    cb, fb = util.oracle_params(net.coarse_bkg_net), util.oracle_params(net.fine_bkg_net)
    H, W = f["hyb_rgb"].shape[:2]
    for can in (1, 0):
        r, d, a = no.render_smpl_nerf(hp, f["h_K"], f["h_c2w"], H, W, b1["verts"], b1["faces"], b1["Ts"], samples_per_ray=24,
                                      render_can=bool(can), geo_threshold=b1["geo_threshold"], interval_comp=0.7)
        assert np.abs(r.reshape(H, W, 3) - f[f"smpl{can}_rgb"]).max() < 1e-5
        assert np.abs(a.reshape(H, W) - f[f"smpl{can}_acc"]).max() < 1e-5
        assert 0 < (f[f"smpl{can}_acc"] > 0).sum() < H * W
    r, d, _ = no.render_hybrid_nerf(cb, fb, hp, f["h_K"], f["h_c2w"], H, W, 0.0, 3.14, b1["verts"], b1["faces"], b1["Ts"],
                                    rays_per_batch=64, samples_per_ray=24, importance_samples_per_ray=16, geo_threshold=b1["geo_threshold"])
    assert np.abs(r.reshape(H, W, 3) - f["hyb_rgb"]).max() < 1e-5 and np.abs(d.reshape(H, W) - f["hyb_depth"]).max() < 5e-5  # depth ~3: batch-size dependent sgemm rounding
    r, d = no.render_hybrid_nerf_multi_persons(cb, fb, [hp, hp], f["h_K"], f["h_c2w"], H, W, 0.0, 3.14,
                                               [b1["verts"], b2["verts"]], [b1["faces"]] * 2, [b1["Ts"], b2["Ts"]],
                                               rays_per_batch=64, samples_per_ray=24, importance_samples_per_ray=16,
                                               geo_threshold=b1["geo_threshold"])
    err = np.abs(r.reshape(H, W, 3) - f["multi_rgb"]).max()
    assert err < 1e-5, err   # same rays_per_batch as the generator: sgemm rounding depends on the batch
