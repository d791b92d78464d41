"""Generates tests/golden/*.npz by running the UNMODIFIED reference (imported from $NEUMAN_REFERENCE,
oracle/ref_import.py) on seeded synthetic inputs.  Run in the build container only:

    python tools/make_golden.py

The GPU box has no reference tree; tests there compare against these committed fixtures.
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import, ref_opts, scenes, synth_smpl      # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def cap_of(ref, K, c2w, H, W, near=0.0, far=3.14):
    cam = ref.pinhole_camera.PinholeCamera(W, H, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    pose = ref.camera_pose.CameraPose.from_camera_to_world(c2w.astype(np.float64))
    cap = ref.captures.BasePinholeCapture(cam, pose)
    cap.near, cap.far = {"bkg": near}, {"bkg": far}
    return cap


def main():
    ref = ref_import.load()
    os.makedirs(OUT, exist_ok=True)
    torch.set_grad_enabled(False)
    g = {}
    # ---------------- stage vectors ----------------
    H, W = 9, 14
    K, c2w = scenes.camera(H, W, seed=3)
    cap = cap_of(ref, K, c2w, H, W)
    g["cam_K"], g["cam_c2w"] = cap.intrinsic_matrix, cap.cam_pose.camera_to_world
    g["cam_HW"] = np.array([H, W])
    xy = np.argwhere(np.ones((H, W)))[:, ::-1]
    g["rays_o0"], g["rays_d0"] = ref.ray_utils.shot_rays(cap, xy)
    o1, d1 = ref.ray_utils.shot_all_rays(cap)
    g["rays_o1"], g["rays_d1"] = o1.astype(np.float32), d1.astype(np.float32)

    torch.manual_seed(0)
    R, S, N = 29, 40, 24
    o = torch.randn(R, 3)
    d = torch.nn.functional.normalize(torch.randn(R, 3), dim=-1) * (0.5 + torch.rand(R, 1))   # non-unit dirs too
    near, far = torch.rand(R, 1), 2 + torch.rand(R, 1)
    batch = {"origin": o, "direction": d, "near": near, "far": far}
    pts, dirs, z = ref.ray_utils.ray_to_samples(batch, S)
    g.update(s_o=o.numpy(), s_d=d.numpy(), s_near=near.numpy(), s_far=far.numpy(), s_pts=pts.numpy(), s_z=z.numpy())
    trand = torch.rand(R, S)
    torch.manual_seed(77)
    trand = torch.rand(R, S)
    torch.manual_seed(77)
    _, _, zp = ref.ray_utils.ray_to_samples(batch, S, perturb=1.0)
    g.update(s_trand=trand.numpy(), s_z_perturb=zp.numpy())
    _, _, zl = ref.ray_utils.ray_to_samples(batch, S, lindisp=True)
    g["s_z_lindisp"] = zl.numpy()
    raw = torch.randn(R, S, 4) * 3
    for wb in (True, False):
        outs = ref.render_utils.raw2outputs(raw, z, d, white_bkg=wb)
        for name, t in zip(("rgb", "disp", "acc", "w", "depth"), outs):
            g[f"c_{name}_{int(wb)}"] = t.numpy()
    g["c_raw"] = raw.numpy()
    w = torch.from_numpy(g["c_w_1"])
    ipts, _, iz = ref.ray_utils.ray_to_importance_samples(batch, z, w, N)
    g.update(i_z=iz.numpy(), i_pts=ipts.numpy())
    _, _, iz2 = ref.ray_utils.ray_to_importance_samples(batch, z, w, N, including_old=False)
    g["i_z_new"] = iz2.numpy()
    bins, wts = torch.sort(torch.rand(R, 17), -1)[0], torch.rand(R, 16)
    u = torch.rand(R, 11)
    torch.manual_seed(5)
    u = torch.rand(R, 11)
    torch.manual_seed(5)
    g.update(p_bins=bins.numpy(), p_w=wts.numpy(), p_u=u.numpy(),
             p_out=ref.ray_utils.sample_pdf(bins, wts, 11, det=False).numpy(),
             p_out_det=ref.ray_utils.sample_pdf(bins, wts, 11, det=True).numpy())
    # near / far
    body = synth_smpl.random_body(seed=2, center=(0.1, 0.0, 0.3))
    Kb, c2wb = scenes.camera(12, 10, focal=16.0, seed=0)
    capb = cap_of(ref, Kb, c2wb, 12, 10)
    ob, db = ref.ray_utils.shot_rays(capb, np.argwhere(np.ones((12, 10)))[:, ::-1])
    nb, fb = ref.ray_utils.geometry_guided_near_far(torch.from_numpy(ob), torch.from_numpy(db),
                                                     torch.from_numpy(body["verts"]), body["geo_threshold"])
    g.update(nf_o=ob, nf_d=db, nf_near=nb.numpy(), nf_far=fb.numpy(), nf_thr=np.float64(body["geo_threshold"]))
    # warp (reference call served by the libigl restatement -- parity unpinned for this stage)
    rng = np.random.RandomState(0)
    wp = (body["verts"].mean(0) + rng.normal(0, 0.12, size=(7, 11, 3))).astype(np.float32)
    cp, cd, cl = ref.ray_utils.warp_samples_to_canonical(wp, body["verts"], np.concatenate([body["faces"]] * 2, 1), body["Ts"])
    g.update(w_pts=wp, w_can=cp.astype(np.float32), w_dirs=cd.astype(np.float32), w_closest=cl.astype(np.float32))
    # networks: seeded default init; golden = reference forward on random inputs
    coarse, fine = scenes.seed_nets(ref.vanilla.build_nerf, ref_opts.default_opt(), 1)
    human, _ = scenes.seed_nets(ref.vanilla.build_nerf, ref_opts.default_opt(posenc="rotate"), 2)
    torch.manual_seed(9)
    npts = torch.randn(300, 3) * 1.5
    nviews = torch.nn.functional.normalize(torch.randn(300, 3), dim=-1)
    g.update(n_pts=npts.numpy(), n_views=nviews.numpy(), n_coarse=coarse(npts, nviews).numpy(),
             n_fine=fine(npts, nviews).numpy(), n_human=human(npts, nviews).numpy(),
             n_sum_coarse=scenes.net_checksum(coarse), n_sum_fine=scenes.net_checksum(fine),
             n_sum_human=scenes.net_checksum(human))
    np.savez_compressed(os.path.join(OUT, "stages.npz"), **g)

    # ---------------- frame renders ----------------
    f = {}
    # BASELINE configs[0]: vanilla background NeRF, 64x64, 64 coarse samples, no fine net
    K, c2w = scenes.camera(64, 64, seed=1)
    cap = cap_of(ref, K, c2w, 64, 64)
    rgb, dep = quiet(ref.render_utils.render_vanilla, coarse, cap, fine_net=None, rays_per_batch=2048,
                     samples_per_ray=64, return_depth=True)
    f.update(cfg1_rgb=rgb, cfg1_depth=dep, cfg1_K=cap.intrinsic_matrix, cfg1_c2w=cap.cam_pose.camera_to_world)
    # coarse + fine, ragged sizes (S, N not multiples of 32)
    K, c2w = scenes.camera(20, 28, seed=2)
    cap = cap_of(ref, K, c2w, 20, 28)
    rgb, dep = quiet(ref.render_utils.render_vanilla, coarse, cap, fine_net=fine, rays_per_batch=100,
                     samples_per_ray=48, importance_samples_per_ray=40, return_depth=True)
    f.update(van_rgb=rgb, van_depth=dep, van_K=cap.intrinsic_matrix, van_c2w=cap.cam_pose.camera_to_world)
    rgb = quiet(ref.render_utils.render_vanilla, coarse, cap, fine_net=fine, rays_per_batch=100,
                samples_per_ray=48, importance_samples_per_ray=40, white_bkg=False)
    f["van_rgb_black"] = rgb
    # human / hybrid / multi-person
    torch.manual_seed(1)
    net = quiet(ref.human_nerf.HumanNeRF, ref_opts.default_opt(num_offset_nets=0))
    scenes.boost_density(net.coarse_human_net)
    f["h_sum"] = np.array([scenes.net_checksum(net.coarse_bkg_net), scenes.net_checksum(net.fine_bkg_net),
                           scenes.net_checksum(net.coarse_human_net)])
    b1 = synth_smpl.random_body(seed=1, center=(0.1, 0.0, 0.3))
    b2 = synth_smpl.random_body(seed=4, center=(-0.15, 0.0, 0.5))
    Hh, Wh = 22, 18
    K, c2w = scenes.camera(Hh, Wh, focal=30.0, seed=0)
    cap = cap_of(ref, K, c2w, Hh, Wh)
    f.update(h_K=cap.intrinsic_matrix, h_c2w=cap.cam_pose.camera_to_world)
    faces = b1["faces"]
    for can in (True, False):
        r, dd, a = quiet(ref.render_utils.render_smpl_nerf, net, cap, b1["verts"], faces, b1["Ts"], rays_per_batch=64,
                         samples_per_ray=24, render_can=can, geo_threshold=b1["geo_threshold"], return_depth=True,
                         return_mask=True, interval_comp=0.7)
        f.update({f"smpl{int(can)}_rgb": r, f"smpl{int(can)}_depth": dd, f"smpl{int(can)}_acc": a})
    r, dd = quiet(ref.render_utils.render_hybrid_nerf, net, cap, b1["verts"], faces, b1["Ts"], rays_per_batch=64,
                  samples_per_ray=24, importance_samples_per_ray=16, geo_threshold=b1["geo_threshold"], return_depth=True)
    f.update(hyb_rgb=r, hyb_depth=dd)
    r, dd = quiet(ref.render_utils.render_hybrid_nerf_multi_persons, net, cap, [net, net], [b1["verts"], b2["verts"]],
                  [faces, faces], [b1["Ts"], b2["Ts"]], rays_per_batch=64, samples_per_ray=24,
                  importance_samples_per_ray=16, geo_threshold=b1["geo_threshold"], return_depth=True)
    f.update(multi_rgb=r, multi_depth=dd)
    np.savez_compressed(os.path.join(OUT, "frames.npz"), **f)
    for n in ("stages.npz", "frames.npz"):
        print(n, os.path.getsize(os.path.join(OUT, n)) // 1024, "KiB")


if __name__ == "__main__":
    main()
