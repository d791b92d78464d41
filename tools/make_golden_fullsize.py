"""Generates tests/golden/fullsize.npz: BASELINE.json configurations 2-5 at their stated sizes, rendered by the
UNMODIFIED reference (imported from $NEUMAN_REFERENCE through oracle/ref_import.py) on one 64x64 pixel block (4096 rays)
per configuration that straddles a body silhouette.  Run in the build container only:

    python tools/make_golden_fullsize.py [cfg2 cfg3 cfg4 cfg5]

The reference's renderers only know whole captures, so the block is rendered through the camera whose principal point
is shifted by the block origin (neuman_b200.synthetic.window_camera): exactly the rays of the full frame's pixels.
Next to every reference output the file stores the measured noise floors on the same rays (SURVEY.md §8d):
  floor64_* : max |fp32 oracle - the same algorithm carried in float64|   (the reference's own rounding noise)
  floor16_* : max |fp32 oracle - fp32 oracle with the MLP's matmul operands rounded to 11 significand bits|
              (what ANY tensor-core evaluation of the nets -- fp16 or tf32 operands -- does to the result)
and `grazing`, the rays whose hit/miss decision or colour is ill-conditioned (|far - near| < 1e-3 for an actor).
"""
import contextlib
import io
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from neuman_b200 import synthetic                                   # noqa: E402
from oracle import neuman_oracle as no                             # noqa: E402
from oracle import ref_import, ref_opts, scenes, synth_smpl        # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fullsize.npz")
WIN = 64


def quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def cap_of(ref, K, c2w, H, W, near, far):
    cam = ref.pinhole_camera.PinholeCamera(W, H, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    pose = ref.camera_pose.CameraPose.from_camera_to_world(c2w.astype(np.float64))
    cap = ref.captures.BasePinholeCapture(cam, pose)
    cap.near, cap.far = {"bkg": near}, {"bkg": far}
    return cap


def pick_window(name, K, c2w, bodies, geo):
    """A 64x64 block with ~half of its rays hitting the first actor (and, for cfg5, a second actor in view if possible)."""
    c = synthetic.FULLSIZE[name]
    H, W = c["H"], c["W"]
    if not bodies:
        return 608, 328                                        # frame centre
    st = 8
    ys, xs = np.meshgrid(np.arange(0, H, st), np.arange(0, W, st), indexing="ij")
    xy = np.stack([xs.reshape(-1), ys.reshape(-1)], 1)
    o, d = no.shot_rays(K, c2w, xy)
    hits = []
    for b in bodies:
        nr, fr = no.geometry_guided_near_far(o, d, b["verts"], geo)
        hits.append((nr < fr).reshape(ys.shape))
    best, arg = -1.0, (0, 0)
    n = WIN // st
    for iy in range(0, ys.shape[0] - n):
        for ix in range(0, ys.shape[1] - n):
            f0 = hits[0][iy:iy + n, ix:ix + n].mean()
            score = 1.0 - abs(f0 - 0.5) * 2
            for h in hits[1:]:
                score += 0.5 * min(h[iy:iy + n, ix:ix + n].mean(), 0.3)
            if score > best:
                best, arg = score, (ix * st, iy * st)
    return arg


def main():
    which = [a for a in sys.argv[1:] if a.startswith("cfg")] or ["cfg2", "cfg3", "cfg4", "cfg5"]
    ref = ref_import.load()
    torch.set_grad_enabled(False)
    out = dict(np.load(OUT)) if os.path.exists(OUT) else {}
    coarse, fine = scenes.seed_nets(ref.vanilla.build_nerf, ref_opts.default_opt(), 1)
    torch.manual_seed(1)
    net = quiet(ref.human_nerf.HumanNeRF, ref_opts.default_opt(num_offset_nets=0))
    scenes.boost_density(net.coarse_human_net)
    out["net_sums"] = np.array([scenes.net_checksum(coarse), scenes.net_checksum(fine), scenes.net_checksum(net.coarse_bkg_net),
                                scenes.net_checksum(net.fine_bkg_net), scenes.net_checksum(net.coarse_human_net)])
    for name in which:
        t0 = time.time()
        c = synthetic.FULLSIZE[name]
        H, W, S, N = c["H"], c["W"], c["S"], c["N"]
        K, c2w = synthetic.fullsize_camera(name)
        bodies = [synth_smpl.random_body(seed=a["seed"], scale=a["scale"], center=a["center"]) for a in c["actors"]]
        geo = bodies[0]["geo_threshold"] if bodies else 0.2
        x0, y0 = pick_window(name, K, c2w, bodies, geo)
        Kw = synthetic.window_camera(K, x0, y0)
        cap = cap_of(ref, Kw, c2w, WIN, WIN, c["near"], c["far"])
        g = {"window": np.array([x0, y0, WIN, WIN]), "geo": np.float64(geo)}
        ru = ref.render_utils
        if name == "cfg2":
            rgb, dep = quiet(ru.render_vanilla, coarse, cap, fine_net=fine, rays_per_batch=2048, samples_per_ray=S,
                             importance_samples_per_ray=N, return_depth=True)
            g.update(rgb=rgb, depth=dep)
            cp, fp = no.net_params_from_joiner(coarse), no.net_params_from_joiner(fine)
            run = lambda: no.render_vanilla(cp, fp, Kw, c2w, WIN, WIN, c["near"], c["far"], rays_per_batch=2048,
                                            samples_per_ray=S, importance_samples_per_ray=N)
        elif name == "cfg3":
            b = bodies[0]
            hp = no.net_params_from_joiner(net.coarse_human_net)
            for can in (1, 0):
                r, d, a = quiet(ru.render_smpl_nerf, net, cap, b["verts"], b["faces"], b["Ts"], rays_per_batch=2048,
                                samples_per_ray=S, render_can=bool(can), geo_threshold=geo, return_depth=True, return_mask=True)
                g.update({f"can{can}_rgb": r, f"can{can}_depth": d, f"can{can}_acc": a})
            run = lambda: no.render_smpl_nerf(hp, Kw, c2w, WIN, WIN, b["verts"], b["faces"], b["Ts"], rays_per_batch=2048,
                                              samples_per_ray=S, render_can=True, geo_threshold=geo)
            # the posed render has its own discontinuities (nearest-triangle flips at the mesh's medial axis move a sample
            # to another part of the canonical body): its floors are measured separately
            run_posed = lambda: no.render_smpl_nerf(hp, Kw, c2w, WIN, WIN, b["verts"], b["faces"], b["Ts"], rays_per_batch=2048,
                                                    samples_per_ray=S, render_can=False, geo_threshold=geo)
        elif name == "cfg4":
            b = bodies[0]
            r, d = quiet(ru.render_hybrid_nerf, net, cap, b["verts"], b["faces"], b["Ts"], rays_per_batch=2048, samples_per_ray=S,
                         importance_samples_per_ray=N, geo_threshold=geo, return_depth=True)
            g.update(rgb=r, depth=d)
            cb, fb, hp = (no.net_params_from_joiner(m) for m in (net.coarse_bkg_net, net.fine_bkg_net, net.coarse_human_net))
            # floors on the background branch + canonical human branch only would miss the merge: run the full driver but
            # reuse the warp results through the (float64) mesh oracle in every precision
            run = lambda: no.render_hybrid_nerf(cb, fb, hp, Kw, c2w, WIN, WIN, c["near"], c["far"], b["verts"], b["faces"], b["Ts"],
                                                rays_per_batch=2048, samples_per_ray=S, importance_samples_per_ray=N,
                                                geo_threshold=geo)[:2]
        else:
            r, d = quiet(ru.render_hybrid_nerf_multi_persons, net, cap, [net] * len(bodies), [b["verts"] for b in bodies],
                         [b["faces"] for b in bodies], [b["Ts"] for b in bodies], rays_per_batch=2048, samples_per_ray=S,
                         importance_samples_per_ray=N, geo_threshold=geo, return_depth=True)
            g.update(rgb=r, depth=d)
            cb, fb, hp = (no.net_params_from_joiner(m) for m in (net.coarse_bkg_net, net.fine_bkg_net, net.coarse_human_net))
            run = lambda: no.render_hybrid_nerf_multi_persons(cb, fb, [hp] * len(bodies), Kw, c2w, WIN, WIN, c["near"], c["far"],
                                                              [b["verts"] for b in bodies], [b["faces"] for b in bodies],
                                                              [b["Ts"] for b in bodies], rays_per_batch=2048, samples_per_ray=S,
                                                              importance_samples_per_ray=N, geo_threshold=geo)
        # grazing rays: an actor's |far - near| below 1e-3 (hit/miss flips under 1-ulp changes; delta_last = 1e10 makes it O(1))
        graz = np.zeros(WIN * WIN, bool)
        if bodies:
            xy = no.all_pixel_coords(WIN, WIN)
            o, d_ = no.shot_rays(Kw, c2w, xy)
            hitany = np.zeros(WIN * WIN, bool)
            for b in bodies:
                nr, fr = no.geometry_guided_near_far(o, d_, b["verts"], geo)
                with np.errstate(invalid="ignore"):
                    graz |= np.isfinite(nr) & (np.abs(fr - nr) < 1e-3)
                hitany |= nr < fr
            g["hit"] = hitany.reshape(WIN, WIN)
        g["grazing"] = graz.reshape(WIN, WIN)
        if name == "cfg3":
            base = run_posed()
            with no.precision(torch.float64):
                hi = run_posed()
            with no.precision(operands="f16"):
                tc = run_posed()
            for k, nm in enumerate(("rgb", "depth", "acc")):
                g[f"posed_floor64_{nm}_map"] = np.abs(base[k] - hi[k]).reshape(WIN * WIN, -1).max(-1).astype(np.float32).reshape(WIN, WIN)
                g[f"posed_floor16_{nm}_map"] = np.abs(base[k] - tc[k]).reshape(WIN * WIN, -1).max(-1).astype(np.float32).reshape(WIN, WIN)
        if run is not None:
            base = run()
            with no.precision(torch.float64):
                hi = run()
            with no.precision(operands="f16"):
                tc = run()
            for k, nm in enumerate(("rgb", "depth", "acc")[:len(base)]):
                d64 = np.abs(base[k] - hi[k]).reshape(WIN * WIN, -1).max(-1)
                d16 = np.abs(base[k] - tc[k]).reshape(WIN * WIN, -1).max(-1)
                g[f"floor64_{nm}"] = np.float64(d64[~graz].max())
                g[f"floor16_{nm}"] = np.float64(d16[~graz].max())
                g[f"floor64_{nm}_map"] = d64.astype(np.float32).reshape(WIN, WIN)    # per ray, for percentile gates
                g[f"floor16_{nm}_map"] = d16.astype(np.float32).reshape(WIN, WIN)
        for k, v in g.items():
            out[f"{name}_{k}"] = v
        print(name, "window", (x0, y0), "hit fraction", float(g["hit"].mean()) if "hit" in g else 0.0, "grazing", int(graz.sum()),
              {k: float(v) for k, v in g.items() if k.startswith("floor") and not k.endswith("_map")}, f"{time.time() - t0:.0f} s", flush=True)
        np.savez_compressed(OUT, **out)
    print(os.path.getsize(OUT) // 1024, "KiB")


if __name__ == "__main__":
    main()
