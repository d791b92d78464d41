"""GPU diagnostic for the MLP kernels: python tools/tc_check.py {simt|tc} [n]
Prints the error of the kernel vs the fp32 oracle and a quick throughput number."""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import neuman_b200 as nb                      # noqa: E402
from neuman_b200 import _lib, ops            # noqa: E402
from oracle import neuman_oracle as no        # noqa: E402
from oracle import scenes                     # noqa: E402

mode_name = sys.argv[1] if len(sys.argv) > 1 else "tc"
n_big = int(sys.argv[2]) if len(sys.argv) > 2 else 4 * 1024 * 1024
mode = {"simt": _lib.NM_MLP_SIMT_F32, "tc": _lib.NM_MLP_TC_F16}[mode_name]
print("mode", mode_name, flush=True)
coarse, fine = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False), 1)
human, _ = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False, posenc="rotate"), 2)
for name, net in (("posenc", coarse), ("rotate", human)):
    p = no.net_params_from_joiner(net)
    net.cuda()
    for n in (128, 256, 1000, 5000):
        torch.manual_seed(n)
        pts, views = torch.randn(n, 3), torch.nn.functional.normalize(torch.randn(n, 3), dim=-1)
        with torch.no_grad():
            ref = no.net_forward(p, pts, views)
        y = ops.joiner_forward(net, pts.cuda(), views.cuda(), mode=mode)
        torch.cuda.synchronize()
        y = y.cpu()
        err = (y - ref).abs()
        print(f"{name} n={n}: max err {err.max().item():.3e} per-channel {err.max(0)[0].tolist()} "
              f"nan {torch.isnan(y).sum().item()} rows>1e-3 {(err.max(1)[0] > 1e-3).sum().item()}", flush=True)
        if err.max() > 1e-2 or torch.isnan(y).any():
            bad = torch.nonzero(err.max(1)[0] > 1e-2).flatten()[:8].tolist()
            print("  first bad rows", bad, "got", y[bad[:2]].tolist() if bad else None, "ref", ref[bad[:2]].tolist() if bad else None)
# throughput
R, S = n_big // 128, 128
o = torch.randn(R, 3, device="cuda") * 0.3
d = torch.nn.functional.normalize(torch.randn(R, 3, device="cuda"), dim=-1)
z = torch.linspace(0, 3.14, S, device="cuda")[None].repeat(R, 1).contiguous()
for it in range(3):
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    raw = ops.mlp_forward_rays(coarse, o, d, z, mode=mode)
    t1.record(); torch.cuda.synchronize()
    ms = t0.elapsed_time(t1)
    print(f"n={R*S}: {ms:.3f} ms  {R*S*1186816/ms/1e9:.1f} TFLOP/s  {R*S/ms/1e3:.2f} Msamples/s", flush=True)
