"""Generates tests/golden/viewless.npz: view-independent nets (NeRF with use_viewdirs=False, the reference's
--use_viewdirs False / --specular_can False) evaluated and rendered by the UNMODIFIED reference, imported from
$NEUMAN_REFERENCE through oracle/ref_import.py (libigl's three hot-path queries are served by the float64 mesh
restatement, as in every generator here).  Run in the build container only:

    NEUMAN_REFERENCE=/path/to/ml-neuman python tools/make_golden_viewless.py

The cases (tests/viewless_cases.py), on the small frames of frames.npz:
  net_{posenc,rotate}_{coarse,fine}  Joiner.forward on the stage inputs of stages.npz (n_pts, n_views)
  van_*                              render_vanilla, view-independent coarse + fine
  smpl{1,0}_*                        render_smpl_nerf of a specular_can=False human, canonical (1) and posed (0)
  hybA_* / hybB_*                    render_hybrid_nerf: view background + view-independent human (A) and the reverse (B)
  multi_*                            render_hybrid_nerf_multi_persons, background of A, humans [A, B]: one actor of each kind
Next to every render, per ray: floor64_* = max |fp32 oracle - float64 oracle| and floor16_* = max |fp32 oracle - oracle
with 11-bit MLP operands| (SURVEY.md §8d), as in make_golden_fullsize.py.  np.savez_compressed is deterministic: a rerun
reproduces the file byte for byte.
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import neuman_oracle as no                             # noqa: E402
from oracle import ref_import, ref_opts, synth_smpl                # noqa: E402
from tests import viewless_cases as vc                             # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "viewless.npz")
GOLD = os.path.join(ROOT, "tests", "golden")


def quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def cap_of(ref, K, c2w, H, W, near, far):
    cam = ref.pinhole_camera.PinholeCamera(W, H, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    pose = ref.camera_pose.CameraPose.from_camera_to_world(np.asarray(c2w).astype(np.float64))
    cap = ref.captures.BasePinholeCapture(cam, pose)
    cap.near, cap.far = {"bkg": near}, {"bkg": far}
    return cap


def floors(out, key, run):
    """Per-ray noise floors of an oracle render `run` () -> (maps...)."""
    base = run()
    with no.precision(torch.float64):
        hi = run()
    with no.precision(operands="f16"):
        tc = run()
    for k, nm in enumerate(("rgb", "depth", "acc")[:len(base)]):
        n = base[k].shape[0] if base[k].ndim > 1 else base[k].size
        out[f"{key}_floor64_{nm}"] = np.abs(base[k] - hi[k]).reshape(n, -1).max(-1).astype(np.float32)
        out[f"{key}_floor16_{nm}"] = np.abs(base[k] - tc[k]).reshape(n, -1).max(-1).astype(np.float32)


def main():
    ref = ref_import.load()
    torch.set_grad_enabled(False)
    stages, frames = np.load(os.path.join(GOLD, "stages.npz")), np.load(os.path.join(GOLD, "frames.npz"))
    out = {}
    # ---- Joiner.forward ----
    pts, views = torch.from_numpy(stages["n_pts"]), torch.from_numpy(stages["n_views"])
    nets = {}
    for pe in ("posenc", "rotate"):
        c, f = vc.viewless_nets(ref.vanilla.build_nerf, ref_opts.default_opt, pe)
        assert type(c).__module__ == "models.vanilla" and not c.nerf.use_viewdirs
        nets[pe] = (c, f)
        for name, j in (("coarse", c), ("fine", f)):
            out[f"net_{pe}_{name}"] = j(pts, views).numpy()
            out[f"net_{pe}_{name}_sum"] = np.float64(vc.checksum(j))
    # ---- render_vanilla ----
    ru = ref.render_utils
    H, W, S, N = vc.VAN["H"], vc.VAN["W"], vc.VAN["S"], vc.VAN["N"]
    K, c2w = frames["van_K"], frames["van_c2w"]
    c, f = nets["posenc"]
    rgb, dep = quiet(ru.render_vanilla, c, cap_of(ref, K, c2w, H, W, 0.0, 3.14), fine_net=f, rays_per_batch=100,
                     samples_per_ray=S, importance_samples_per_ray=N, return_depth=True)
    out.update(van_rgb=rgb, van_depth=dep)
    cp, fp = no.net_params_from_joiner(c), no.net_params_from_joiner(f)
    floors(out, "van", lambda: no.render_vanilla(cp, fp, K, c2w, H, W, 0.0, 3.14, samples_per_ray=S, importance_samples_per_ray=N))
    # ---- human renderers ----
    H, W, S, N = vc.HUM["H"], vc.HUM["W"], vc.HUM["S"], vc.HUM["N"]
    K, c2w = frames["h_K"], frames["h_c2w"]
    cap = cap_of(ref, K, c2w, H, W, 0.0, 3.14)
    b1 = synth_smpl.random_body(seed=1, center=(0.1, 0.0, 0.3))
    b2 = synth_smpl.random_body(seed=4, center=(-0.15, 0.0, 0.5))
    geo = b1["geo_threshold"]
    models = {k: quiet(vc.human_model, ref.human_nerf.HumanNeRF, ref_opts.default_opt, k) for k in vc.HUMANS}
    for k, m in models.items():
        out[f"human{k}_sums"] = np.array([vc.checksum(m.coarse_bkg_net), vc.checksum(m.fine_bkg_net), vc.checksum(m.coarse_human_net)])
    params = {k: [no.net_params_from_joiner(j) for j in (m.coarse_bkg_net, m.fine_bkg_net, m.coarse_human_net)]
              for k, m in models.items()}
    A = models["A"]
    assert not A.coarse_human_net.nerf.use_viewdirs and not models["B"].coarse_bkg_net.nerf.use_viewdirs
    for can in (1, 0):
        r, d, a = quiet(ru.render_smpl_nerf, A, cap, b1["verts"], b1["faces"], b1["Ts"], rays_per_batch=64, samples_per_ray=S,
                        render_can=bool(can), geo_threshold=geo, return_depth=True, return_mask=True)
        out.update({f"smpl{can}_rgb": r, f"smpl{can}_depth": d, f"smpl{can}_acc": a})
        hp = params["A"][2]
        floors(out, f"smpl{can}", lambda: no.render_smpl_nerf(hp, K, c2w, H, W, b1["verts"], b1["faces"], b1["Ts"], samples_per_ray=S,
                                                              render_can=bool(can), geo_threshold=geo))
    for k, m in models.items():
        r, d = quiet(ru.render_hybrid_nerf, m, cap, b1["verts"], b1["faces"], b1["Ts"], rays_per_batch=64, samples_per_ray=S,
                     importance_samples_per_ray=N, geo_threshold=geo, return_depth=True)
        out.update({f"hyb{k}_rgb": r, f"hyb{k}_depth": d})
        cb, fb, hp = params[k]
        floors(out, f"hyb{k}", lambda: no.render_hybrid_nerf(cb, fb, hp, K, c2w, H, W, 0.0, 3.14, b1["verts"], b1["faces"], b1["Ts"],
                                                             samples_per_ray=S, importance_samples_per_ray=N, geo_threshold=geo)[:2])
    bodies = [b1, b2]
    r, d = quiet(ru.render_hybrid_nerf_multi_persons, A, cap, [A, models["B"]], [b["verts"] for b in bodies],
                 [b["faces"] for b in bodies], [b["Ts"] for b in bodies], rays_per_batch=64, samples_per_ray=S,
                 importance_samples_per_ray=N, geo_threshold=geo, return_depth=True)
    out.update(multi_rgb=r, multi_depth=d)
    cb, fb = params["A"][:2]
    hs = [params["A"][2], params["B"][2]]
    floors(out, "multi", lambda: no.render_hybrid_nerf_multi_persons(cb, fb, hs, K, c2w, H, W, 0.0, 3.14,
                                                                     [b["verts"] for b in bodies], [b["faces"] for b in bodies],
                                                                     [b["Ts"] for b in bodies], samples_per_ray=S,
                                                                     importance_samples_per_ray=N, geo_threshold=geo))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT) // 1024, "KiB", {k: float(np.max(v)) for k, v in out.items() if "floor" in k})


if __name__ == "__main__":
    main()
