"""View-dependent vs view-independent nets (use_viewdirs=False) on the same frames, alternating:

    python tools/viewless_bench.py [rounds]        # default 3 rounds of each kind per workload

Workloads: render_vanilla 1280x720 with 128 + 128 samples (bench.py's flagship frame), and the hybrid configuration
(BASELINE cfg4: render_hybrid_nerf 1280x720, 128 + 128, one actor) where both background nets and the canonical human net
are of the kind under test.  Every round renders one warm-up frame and one timed frame per kind; the MLP launches of the
timed frame are bracketed by CUDA events (nm_profile_*).  Prints per kind: Mrays/s, MLP ms per frame, MLP evaluations per
frame and MLP TFLOP/s counted with 1 186 816 (view-dependent) / 984 064 (view-independent) FLOP per evaluation, and the
median over the rounds; then the GPU name and its power limit (nvidia-smi; the rate depends on it)."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import neuman_b200 as nb                                            # noqa: E402
from neuman_b200 import ops, render, synthetic                      # noqa: E402
from tests import viewless_cases as vc                              # noqa: E402

FLOP = {"view": 1186816, "viewless": 984064}


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        return r.stdout.strip() + " W"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def human_model(viewless):
    """HumanNeRF with all three nets of one kind (seeded as bench.py's / tests/viewless_cases.py's)."""
    torch.manual_seed(1)
    m = nb.HumanNeRF(nb.default_opt(use_cuda=False, use_viewdirs=not viewless, specular_can=not viewless))
    if viewless:
        for j in (m.coarse_bkg_net, m.fine_bkg_net, m.coarse_human_net):
            vc.boost_viewless(j)
    else:
        synthetic.boost_density(m.coarse_human_net)
    return m.cuda()


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    torch.set_grad_enabled(False)
    ctx = ops.Context.get(0)
    cfg = synthetic.FULLSIZE["cfg4"]
    H, W, S, N = cfg["H"], cfg["W"], cfg["S"], cfg["N"]
    K, c2w = synthetic.fullsize_camera("cfg4")
    cap = nb.SimpleCapture(K, c2w, H, W, cfg["near"], cfg["far"])
    sm = synthetic.make_model(0)
    par = sm["kintree_table"][0].astype(np.int64)
    smpl = ops.SmplModelDevice(sm["v_template"], sm["shapedirs"], sm["J_regressor"], sm["weights"], par, device="cuda")
    faces = torch.from_numpy(sm["f"].astype(np.int32)).cuda()
    a = cfg["actors"][0]
    pose, betas, align = synthetic.actor_pose(a)
    verts, joints, T = ops.smpl_scene_transforms(smpl, pose, betas, align, a["scale"])
    geo = float(torch.linalg.norm(joints[3] - joints[0]))
    models = {"view": human_model(False), "viewless": human_model(True)}
    work = {
        "vanilla": lambda m: render.render_vanilla_range(m.coarse_bkg_net, cap, m.fine_bkg_net, S, N, pix0=0, n=H * W,
                                                         host_out=False),
        "hybrid": lambda m: render.render_hybrid_nerf_range(m, cap, verts.contiguous(), faces, T, S, N, True, geo, pix0=0,
                                                            n=H * W, host_out=False),
    }
    res = {(w, k): [] for w in work for k in models}
    for r in range(rounds):
        for w, fn in work.items():
            for k, m in models.items():
                fn(m)                                                   # warm-up (packing, workspace)
                torch.cuda.synchronize()
                ctx.profile(True)
                t0 = time.perf_counter()
                fn(m)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                p = ctx.profile_read()
                ctx.profile(False)
                tflops = p["mlp_evals"] * FLOP[k] / (p["mlp_ms"] * 1e-3) / 1e12
                res[(w, k)].append((H * W / dt / 1e6, p["mlp_ms"], p["mlp_evals"], tflops))
                print(f"round {r} {w:8s} {k:9s} {H * W / dt / 1e6:7.3f} Mrays/s  MLP {p['mlp_ms']:8.2f} ms/frame  "
                      f"{p['mlp_evals'] / 1e6:7.2f} M evals  {tflops:6.1f} TFLOP/s", flush=True)
    print("median over", rounds, "rounds:")
    for (w, k), v in res.items():
        v = np.array(v)
        med = np.median(v, 0)
        print(f"  {w:8s} {k:9s} {med[0]:7.3f} Mrays/s  MLP {med[1]:8.2f} ms/frame  {med[3]:6.1f} TFLOP/s  "
              f"MLP time per evaluation {med[1] / med[2] * 1e6:.3f} ns")
    print("GPU:", torch.cuda.get_device_name(0), "power limit:", power_limit())


if __name__ == "__main__":
    main()
