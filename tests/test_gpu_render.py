"""GPU parity of the frame drivers against the reference goldens (small frames) and the oracle, plus
size-independent properties at BASELINE.json's full frame sizes."""
import numpy as np
import pytest
import torch

import neuman_b200 as nb
from neuman_b200 import render
from oracle import neuman_oracle as no
from oracle import scenes
from tests import util

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-4         # north_star: rendered RGB / depth <= 1e-4 abs vs the reference path (fp32)


@pytest.fixture(scope="module")
def nets():
    return tuple(n.to(DEV) for n in util.product_nets())


@pytest.fixture(scope="module")
def human():
    return util.product_human_model(DEV)


def test_cfg1_vanilla_64x64(nets):
    """BASELINE configs[0]: vanilla background NeRF, 64x64, 64 coarse samples."""
    f = util.golden("frames.npz")
    cap = nb.SimpleCapture(f["cfg1_K"], f["cfg1_c2w"], 64, 64, 0.0, 3.14)
    rgb, dep = nb.render_vanilla(nets[0], cap, fine_net=None, samples_per_ray=64, return_depth=True)
    assert rgb.dtype == np.float32 and rgb.shape == (64, 64, 3) and dep.shape == (64, 64)
    assert np.abs(rgb - f["cfg1_rgb"]).max() < TOL and np.abs(dep - f["cfg1_depth"]).max() < TOL
    assert round(util.psnr(rgb, f["cfg1_rgb"]), 2) >= 70.0


def test_vanilla_coarse_fine_ragged(nets):
    f = util.golden("frames.npz")
    cap = nb.SimpleCapture(f["van_K"], f["van_c2w"], 20, 28, 0.0, 3.14)
    rgb, dep = nb.render_vanilla(nets[0], cap, fine_net=nets[1], samples_per_ray=48, importance_samples_per_ray=40,
                                 return_depth=True)
    cp, fp = (util.oracle_params(m.to("cpu")) for m in nets[:2])
    for m in nets:
        m.to(DEV)
    fl = util.floors16(lambda: no.render_vanilla(cp, fp, f["van_K"], f["van_c2w"], 20, 28, 0.0, 3.14, samples_per_ray=48,
                                                 importance_samples_per_ray=40))
    e_rgb, e_dep = np.abs(rgb - f["van_rgb"]).max(), np.abs(dep - f["van_depth"]).max()
    assert e_rgb < TOL and e_dep <= util.gate(e_dep, fl[1]), (e_rgb, e_dep, fl)
    rgb = nb.render_vanilla(nets[0], cap, fine_net=nets[1], samples_per_ray=48, importance_samples_per_ray=40, white_bkg=False)
    assert np.abs(rgb - f["van_rgb_black"]).max() < TOL


def test_human_renderers_golden(human):
    f = util.golden("frames.npz")
    b1, b2 = util.bodies()
    H, W = f["hyb_rgb"].shape[:2]
    cap = nb.SimpleCapture(f["h_K"], f["h_c2w"], H, W, 0.0, 3.14)
    geo = b1["geo_threshold"]

    def close(a, ref, tol, what):
        err = np.abs(a - ref)
        # grazing rays (hit/miss decided by an ill-conditioned sqrt) may flip: allow <1% outlier pixels
        bad = (err > tol).reshape(H * W, -1).any(-1).mean()
        assert bad < 0.01, (what, bad, err.max())

    for can in (1, 0):
        r, d, a = nb.render_smpl_nerf(human, cap, b1["verts"], b1["faces"], b1["Ts"], samples_per_ray=24,
                                      render_can=bool(can), geo_threshold=geo, return_depth=True, return_mask=True,
                                      interval_comp=0.7)
        close(r, f[f"smpl{can}_rgb"], TOL, f"smpl{can} rgb")
        close(d, f[f"smpl{can}_depth"], TOL, f"smpl{can} depth")
        close(a, f[f"smpl{can}_acc"], TOL, f"smpl{can} acc")
    r, d = nb.render_hybrid_nerf(human, cap, b1["verts"], b1["faces"], b1["Ts"], samples_per_ray=24,
                                 importance_samples_per_ray=16, geo_threshold=geo, return_depth=True)
    cb, fb, hp = (util.oracle_params(m.to("cpu")) for m in (human.coarse_bkg_net, human.fine_bkg_net, human.coarse_human_net))
    human.to(DEV)
    fl_h = util.floors16(lambda: no.render_hybrid_nerf(cb, fb, hp, f["h_K"], f["h_c2w"], H, W, 0.0, 3.14, b1["verts"], b1["faces"],
                                                       b1["Ts"], samples_per_ray=24, importance_samples_per_ray=16,
                                                       geo_threshold=geo)[:2])
    close(r, f["hyb_rgb"], util.gate(0, fl_h[0]), "hybrid rgb")
    close(d, f["hyb_depth"], util.gate(0, fl_h[1]), "hybrid depth")
    r, d = nb.render_hybrid_nerf_multi_persons(human, cap, [human, human], [b1["verts"], b2["verts"]],
                                               [b1["faces"]] * 2, [b1["Ts"], b2["Ts"]], samples_per_ray=24,
                                               importance_samples_per_ray=16, geo_threshold=geo, return_depth=True)
    fl_m = util.floors16(lambda: no.render_hybrid_nerf_multi_persons(cb, fb, [hp, hp], f["h_K"], f["h_c2w"], H, W, 0.0, 3.14,
                                                                     [b1["verts"], b2["verts"]], [b1["faces"]] * 2,
                                                                     [b1["Ts"], b2["Ts"]], samples_per_ray=24,
                                                                     importance_samples_per_ray=16, geo_threshold=geo))
    close(r, f["multi_rgb"], util.gate(0, fl_m[0]), "multi rgb")
    close(d, f["multi_depth"], util.gate(0, fl_m[1]), "multi depth")


def test_full_size_properties(nets):
    """1280x720, 128+128 (the benchmark workload): results do not depend on the device chunking or on
    how the frame is sharded into pixel ranges; white-vs-black background differ by exactly 1-acc; a
    4096-ray subsample agrees with the oracle."""
    H, W = 720, 1280
    K, c2w = scenes.camera(H, W, seed=1)
    cap = nb.SimpleCapture(K, c2w, H, W, 0.0, 3.14)
    n = H * W
    sub0, cnt = 300 * W + 17, 6000
    a_rgb, a_dep = render.render_vanilla_range(nets[0], cap, nets[1], 128, 128, pix0=sub0, n=cnt, host_out=False)
    b_rgb, b_dep = render.render_vanilla_range(nets[0], cap, nets[1], 128, 128, pix0=sub0, n=cnt, host_out=False, chunk=1000)
    assert torch.equal(a_rgb, b_rgb) and torch.equal(a_dep, b_dep)               # chunk-invariant
    c_rgb, _ = render.render_vanilla_range(nets[0], cap, nets[1], 128, 128, pix0=sub0 + 1000, n=2000, host_out=False)
    assert torch.equal(c_rgb, a_rgb[1000:3000])                                  # shard-invariant
    k_rgb, _ = render.render_vanilla_range(nets[0], cap, nets[1], 128, 128, white_bkg=False, pix0=sub0, n=cnt, host_out=False)
    assert ((a_rgb - k_rgb) >= -1e-6).all() and ((a_rgb - k_rgb) <= 1 + 1e-6).all()
    # oracle on the first 1024 rays of the range
    idx = np.arange(sub0, sub0 + 1024)
    cp, fp = (util.oracle_params(m.to("cpu")) for m in nets[:2])
    for m in nets:
        m.to(DEV)
    rgb_o, dep_o = no.render_vanilla(cp, fp, K, c2w, H, W, 0.0, 3.14, samples_per_ray=128, importance_samples_per_ray=128,
                                     ray_subset=idx)
    rgb = a_rgb[:1024].cpu().numpy()
    fl = util.floors16(lambda: no.render_vanilla(cp, fp, K, c2w, H, W, 0.0, 3.14, samples_per_ray=128, importance_samples_per_ray=128,
                                                 ray_subset=idx))
    e_dep = np.abs(a_dep[:1024].cpu().numpy() - dep_o).max()
    assert np.abs(rgb - rgb_o).max() < TOL and e_dep <= util.gate(e_dep, fl[1]), (e_dep, fl)
    assert abs(round(util.psnr(rgb, 0.5 * np.ones_like(rgb)), 2) - round(util.psnr(rgb_o, 0.5 * np.ones_like(rgb)), 2)) <= 0.01
    # BASELINE configs[1]: the same frame at 64 + 128 samples
    c_rgb, c_dep = render.render_vanilla_range(nets[0], cap, nets[1], 64, 128, pix0=sub0, n=1024, host_out=True)
    rgb_o, dep_o = no.render_vanilla(cp, fp, K, c2w, H, W, 0.0, 3.14, samples_per_ray=64, importance_samples_per_ray=128,
                                     ray_subset=idx)
    fl = util.floors16(lambda: no.render_vanilla(cp, fp, K, c2w, H, W, 0.0, 3.14, samples_per_ray=64, importance_samples_per_ray=128,
                                                 ray_subset=idx))
    e_dep = np.abs(c_dep.numpy() - dep_o).max()
    assert np.abs(c_rgb.numpy() - rgb_o).max() < TOL and e_dep <= util.gate(e_dep, fl[1]), (e_dep, fl)


def test_human_shard_chunk_invariance_and_determinism(human):
    """Hit rays are compacted with atomics (order varies run to run): results must not depend on it, nor on
    the device chunk size or the pixel range the frame is sharded into."""
    b1, b2 = util.bodies()
    H, W = 96, 128
    K, c2w = scenes.camera(H, W, focal=110.0, seed=0)
    cap = nb.SimpleCapture(K, c2w, H, W, 0.0, 3.14)
    geo = b1["geo_threshold"]
    full = render.render_hybrid_nerf_range(human, cap, b1["verts"], b1["faces"], b1["Ts"], 32, 32, True, geo, host_out=False)
    again = render.render_hybrid_nerf_range(human, cap, b1["verts"], b1["faces"], b1["Ts"], 32, 32, True, geo, host_out=False)
    small = render.render_hybrid_nerf_range(human, cap, b1["verts"], b1["faces"], b1["Ts"], 32, 32, True, geo, host_out=False,
                                            chunk=777)
    for a, b, c in zip(full, again, small):
        assert torch.equal(a, b) and torch.equal(a, c)
    assert 0 < int((full[2] > 0).sum()) < H * W                      # hits and misses both present
    p0, n = 3000, 5000
    part = render.render_hybrid_nerf_range(human, cap, b1["verts"], b1["faces"], b1["Ts"], 32, 32, True, geo, pix0=p0, n=n,
                                           host_out=True)
    for a, b in zip(full, part):
        assert torch.equal(a[p0:p0 + n].cpu(), b)
    # multi-person: shard invariance through the public function (pix0 / n)
    m_full = nb.render_hybrid_nerf_multi_persons(human, cap, [human, human], [b1["verts"], b2["verts"]], [b1["faces"]] * 2,
                                                 [b1["Ts"], b2["Ts"]], samples_per_ray=32, importance_samples_per_ray=32,
                                                 geo_threshold=geo)
    m_part = nb.render_hybrid_nerf_multi_persons(human, cap, [human, human], [b1["verts"], b2["verts"]], [b1["faces"]] * 2,
                                                 [b1["Ts"], b2["Ts"]], samples_per_ray=32, importance_samples_per_ray=32,
                                                 geo_threshold=geo, pix0=p0, n=n)
    assert np.array_equal(m_full.reshape(-1, 3)[p0:p0 + n], m_part)
    # chunk invariance of the human-only and the multi-person drivers
    s_full = render.render_smpl_nerf_range(human, cap, b1["verts"], b1["faces"], b1["Ts"], 32, True, False, geo, 1.0, host_out=False)
    s_small = render.render_smpl_nerf_range(human, cap, b1["verts"], b1["faces"], b1["Ts"], 32, True, False, geo, 1.0, host_out=False,
                                            chunk=777)
    m_dev, m_small = (render._hybrid(human, [human, human], cap, [b1["verts"], b2["verts"]], [b1["faces"]] * 2, [b1["Ts"], b2["Ts"]],
                                     32, 32, True, geo, True, 0, None, False, chunk) for chunk in (render.CHUNK, 777))
    for a, b in zip(s_full + m_dev, s_small + m_small):
        assert torch.equal(a, b)
    assert np.array_equal(m_full.reshape(-1, 3), m_dev[0].cpu().numpy())


def test_human_all_miss_frame(human):
    """Camera looking away from the body: every ray misses -> white / zero maps for render_smpl_nerf, the
    background composite for the hybrid renderers (acc = 0 everywhere)."""
    b1, _ = util.bodies()
    H, W = 24, 32
    K, c2w = scenes.camera(H, W, focal=40.0, seed=0, yaw=1.5708)      # looks along +x: every ray passes >1 unit from the body
    # (a camera turned fully away would still "hit": the reference accepts spheres behind the origin, near<far<0)
    cap = nb.SimpleCapture(K, c2w, H, W, 0.0, 3.14)
    r, d, a = nb.render_smpl_nerf(human, cap, b1["verts"], b1["faces"], b1["Ts"], samples_per_ray=16,
                                  geo_threshold=b1["geo_threshold"], return_depth=True, return_mask=True)
    assert (r == 1.0).all() and (d == 0).all() and (a == 0).all()
    r0 = nb.render_smpl_nerf(human, cap, b1["verts"], b1["faces"], b1["Ts"], samples_per_ray=16, white_bkg=False,
                             geo_threshold=b1["geo_threshold"])
    assert (r0 == 0.0).all()
    rh, dh, ah = render.render_hybrid_nerf_range(human, cap, b1["verts"], b1["faces"], b1["Ts"], 32, 32, True,
                                                 b1["geo_threshold"], host_out=True)
    assert (ah == 0).all()
    cb, fb = (util.oracle_params(m.to("cpu")) for m in (human.coarse_bkg_net, human.fine_bkg_net))
    human.to(DEV)
    hp = util.oracle_params(human.coarse_human_net.to("cpu"))
    human.to(DEV)
    ro, do_, _ = no.render_hybrid_nerf(cb, fb, hp, K, c2w, H, W, 0.0, 3.14, b1["verts"], b1["faces"], b1["Ts"],
                                       samples_per_ray=32, importance_samples_per_ray=32, geo_threshold=b1["geo_threshold"])
    # few coarse samples make sample_pdf's `denom < 1e-5` discontinuity visible on isolated rays: allow 1 % outliers
    fl = util.floors16(lambda: no.render_hybrid_nerf(cb, fb, hp, K, c2w, H, W, 0.0, 3.14, b1["verts"], b1["faces"], b1["Ts"],
                                                     samples_per_ray=32, importance_samples_per_ray=32,
                                                     geo_threshold=b1["geo_threshold"])[:2])
    bad = (np.abs(rh.numpy() - ro).max(-1) > util.gate(0, fl[0])) | (np.abs(dh.numpy() - do_) > util.gate(0, fl[1]))
    assert bad.mean() < 0.01, (bad.mean(), np.abs(rh.numpy() - ro).max())
