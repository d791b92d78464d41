"""NeRF-T nets (position input (x, y, z, t), --ablate_nerft) vs plain view-dependent nets on the same frame, alternating:

    python tools/nerft_bench.py [rounds]        # default 3 rounds of each kind

Workload: render_vanilla 1280x720 with 128 + 128 samples (bench.py's flagship frame; the NeRF-T kind renders it with
ablate_nerft at frame 7 of 30).  Every round renders one warm-up frame and one timed frame per kind; the MLP launches of the
timed frame are bracketed by CUDA events (nm_profile_*).  Prints per kind: Mrays/s, MLP ms per frame, MLP evaluations per
frame and MLP TFLOP/s counted with 1 186 816 (plain) / 1 208 320 (NeRF-T: 84-wide layers 0 and 5) FLOP per evaluation, and
the median over the rounds.  Then the background trainer's step (train.train_batch: 2048 rays, 128 + 128 samples, Adam;
the NeRF-T kind with opt.ablate_nerft and per-ray times from 4 frames), 20 steps per kind and round after 3 warm-up steps,
timed with a device synchronise; then the GPU name and its power limit (nvidia-smi; the rate depends on it)."""
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

FLOP = {"plain": 1186816, "nerft": 1208320}


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        return r.stdout.strip() + " W"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def nets(nerft):
    torch.manual_seed(1)
    c, f = nb.build_nerf(nb.default_opt(use_cuda=False, raw_pos_dim=4 if nerft else 3))
    for j in (c, f):
        synthetic.boost_density(j)
    return c.cuda(), f.cuda()


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    torch.set_grad_enabled(False)
    ctx = ops.Context.get(0)
    cfg = synthetic.FULLSIZE["cfg4"]
    H, W, S, N = cfg["H"], cfg["W"], cfg["S"], cfg["N"]
    K, c2w = synthetic.fullsize_camera("cfg4")
    cap = nb.SimpleCapture(K, c2w, H, W, cfg["near"], cfg["far"])
    kinds = {"plain": (nets(False), None), "nerft": (nets(True), float(np.float32(7 / 30)))}
    res = {k: [] for k in kinds}
    for r in range(rounds):
        for k, ((c, f), t) in kinds.items():
            def frame():
                return render.render_vanilla_range(c, cap, f, S, N, pix0=0, n=H * W, host_out=False, frame_time=t)
            frame()                                                 # warm-up (packing, workspace)
            torch.cuda.synchronize()
            ctx.profile(True)
            t0 = time.perf_counter()
            frame()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            p = ctx.profile_read()
            ctx.profile(False)
            tflops = p["mlp_evals"] * FLOP[k] / (p["mlp_ms"] * 1e-3) / 1e12
            res[k].append((H * W / dt / 1e6, p["mlp_ms"], p["mlp_evals"], tflops))
            print(f"round {r} {k:6s} {H * W / dt / 1e6:7.3f} Mrays/s  MLP {p['mlp_ms']:8.2f} ms/frame  "
                  f"{p['mlp_evals'] / 1e6:7.2f} M evals  {tflops:6.1f} TFLOP/s", flush=True)
    print("median over", rounds, "rounds:")
    for k, v in res.items():
        med = np.median(np.array(v), 0)
        print(f"  {k:6s} {med[0]:7.3f} Mrays/s  MLP {med[1]:8.2f} ms/frame  {med[3]:6.1f} TFLOP/s  "
              f"MLP time per evaluation {med[1] / med[2] * 1e6:.3f} ns")
    # ---- training step ----
    from neuman_b200 import train as nt
    torch.set_grad_enabled(True)
    R, steps = 2048, 20
    g = torch.Generator().manual_seed(3)
    batch = dict(origin=(torch.randn(R, 3, generator=g) * 0.1).cuda(),
                 direction=torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1).cuda(),
                 near=torch.full((R,), 0.5, device="cuda"), far=torch.full((R,), 4.0, device="cuda"),
                 color=torch.rand(R, 3, generator=g).cuda(), depth=(1.5 + torch.rand(R, generator=g)).cuda(),
                 viewf_list=torch.tensor([7 / 30, 11 / 30, 19 / 30, 29 / 30]).repeat_interleave(R // 4)[:, None].cuda())
    tres = {k: [] for k in kinds}
    for r in range(rounds):
        for k, ((c, f), _) in kinds.items():
            opt = nb.default_opt(samples_per_ray=128, importance_samples_per_ray=128, perturb=1.0, raw_noise_std=1.0,
                                 ablate_nerft=k == "nerft")
            optim = torch.optim.Adam(list(c.parameters()) + list(f.parameters()), lr=5e-4)
            for it in range(3):
                nt.train_batch(c, f, optim, batch, opt, iteration=it, check_bad_weights=False)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for it in range(steps):
                nt.train_batch(c, f, optim, batch, opt, iteration=it, check_bad_weights=False)
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) / steps * 1e3
            tres[k].append(ms)
            print(f"round {r} train step {k:6s} {ms:7.2f} ms", flush=True)
    for k, v in tres.items():
        print(f"  train step {k:6s} median {np.median(v):7.2f} ms")
    print("GPU:", torch.cuda.get_device_name(0), "power limit:", power_limit())


if __name__ == "__main__":
    main()
