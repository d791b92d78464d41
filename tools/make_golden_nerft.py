"""Generates tests/golden/nerft.npz: NeRF-T nets (the reference's --ablate_nerft background nets, position input
(x, y, z, t), train.py:254-256) evaluated and rendered by the UNMODIFIED reference, imported from $NEUMAN_REFERENCE through
oracle/ref_import.py.  Run in the build container only:

    NEUMAN_REFERENCE=/path/to/ml-neuman python tools/make_golden_nerft.py

The cases (tests/nerft_cases.py):
  pts, views, net_{coarse,fine}  Joiner.forward on the stage samples of stages.npz with a time column (0, 1, k/30, random),
                                 then 50 of them at two times
  van{0,1}_*                     render_vanilla(ablate_nerft=True) of the coarse + fine nets on frames.npz's vanilla camera
                                 at frame_id / total_frames = FRAMES[0], FRAMES[1]
Next to every render, per ray: floor64_* = max |fp32 oracle - float64 oracle| and floor16_* = max |fp32 oracle - oracle
with 11-bit MLP operands| (SURVEY.md §8d), as in make_golden_viewless.py.  np.savez_compressed is deterministic: a rerun
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
from oracle import ref_import, ref_opts                            # noqa: E402
from tests import nerft_cases as nc                                # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "nerft.npz")
GOLD = os.path.join(ROOT, "tests", "golden")


def main():
    ref = ref_import.load()
    torch.set_grad_enabled(False)
    stages, frames = np.load(os.path.join(GOLD, "stages.npz")), np.load(os.path.join(GOLD, "frames.npz"))
    c, f = nc.nerft_nets(ref.vanilla.build_nerf, ref_opts.default_opt)
    assert type(c).__module__ == "models.vanilla" and c.pos_pe.input_dims == 4 and c.nerf.pts_linears[0].weight.shape[1] == 84
    pts, views = nc.net_inputs(stages)
    out = dict(pts=pts, views=views)
    for name, j in (("coarse", c), ("fine", f)):
        out[f"net_{name}"] = j(torch.from_numpy(pts), torch.from_numpy(views)).numpy()
    H, W, S, N = nc.VAN["H"], nc.VAN["W"], nc.VAN["S"], nc.VAN["N"]
    K, c2w = frames["van_K"], frames["van_c2w"]
    cp, fp = no.net_params_from_joiner(c), no.net_params_from_joiner(f)
    for i, (fid, total) in enumerate(nc.FRAMES):
        cam = ref.pinhole_camera.PinholeCamera(W, H, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
        cap = ref.captures.BasePinholeCapture(cam, ref.camera_pose.CameraPose.from_camera_to_world(np.asarray(c2w).astype(np.float64)))
        cap.near, cap.far = {"bkg": nc.NEAR}, {"bkg": nc.FAR}
        cap.frame_id = {"frame_id": fid, "total_frames": total}
        with contextlib.redirect_stdout(io.StringIO()):
            rgb, dep = ref.render_utils.render_vanilla(c, cap, fine_net=f, rays_per_batch=100, samples_per_ray=S,
                                                       importance_samples_per_ray=N, return_depth=True, ablate_nerft=True)
        out.update({f"van{i}_rgb": rgb, f"van{i}_depth": dep})
        t = nc.frame_time(fid, total)
        base = nc.oracle_render(cp, fp, K, c2w, H, W, t)
        with no.precision(torch.float64):
            hi = nc.oracle_render(cp, fp, K, c2w, H, W, t)
        with no.precision(operands="f16"):
            tc = nc.oracle_render(cp, fp, K, c2w, H, W, t)
        for k, nm in enumerate(("rgb", "depth")):
            n = base[k].shape[0]
            out[f"van{i}_floor64_{nm}"] = np.abs(base[k] - hi[k]).reshape(n, -1).max(-1).astype(np.float32)
            out[f"van{i}_floor16_{nm}"] = np.abs(base[k] - tc[k]).reshape(n, -1).max(-1).astype(np.float32)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT) // 1024, "KiB", {k: float(np.max(v)) for k, v in out.items() if "floor" in k})


if __name__ == "__main__":
    main()
