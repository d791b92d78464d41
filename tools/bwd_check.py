"""GPU diagnostic for the backward chain kernel: python tools/bwd_check.py [n]
Compares every intermediate gradient plane of k_mlp_tc_bwd with the torch restatement on the same stash
(tests/util.py: chain_torch, put in place of neuman_b200.autograd._chain_kernel for the second pass)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import neuman_b200 as nb                      # noqa: E402
from neuman_b200 import autograd as nag       # noqa: E402
from tests.util import chain_torch            # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 3000
coarse, _ = nb.build_nerf(nb.default_opt())
torch.manual_seed(0)
pts = torch.randn(n, 3, device="cuda") * 1.5
views = torch.nn.functional.normalize(torch.randn(n, 3, device="cuda"), dim=-1)
g = torch.randn(n, 4, device="cuda")
cap = {}
orig = nag._weight_grads
kernel_chain = nag._chain_kernel


def spy(joiner, stash, pts_, views_, gg, g_pre, g_f, g_v, inv):
    cap[nag._chain_kernel is kernel_chain] = (g_pre.float() * inv, g_f.float() * inv, g_v.float() * inv)
    return orig(joiner, stash, pts_, views_, gg, g_pre, g_f, g_v, inv)


nag._weight_grads = spy
for chain in (kernel_chain, chain_torch):
    nag._chain_kernel = chain
    coarse.zero_grad()
    raw = coarse(pts, views)
    (raw * g).sum().backward()
    torch.cuda.synchronize()
k, t = cap[True], cap[False]


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


print("g_v", rel(k[2], t[2]), "g_f", rel(k[1], t[1]))
for l in range(7, -1, -1):
    d = (k[0][l] - t[0][l]).abs()
    print(f"g_pre[{l}] rel {rel(k[0][l], t[0][l]):.3e} max abs {float(d.max()):.3e} ref max {float(t[0][l].abs().max()):.3e} "
          f"bad rows {int((d.max(1)[0] > 1e-2 * t[0][l].abs().max()).sum())} nan {int(torch.isnan(k[0][l]).sum())}")
    if l == 7:
        bad = torch.nonzero(d.max(1)[0] > 1e-2 * t[0][l].abs().max()).flatten()[:10].tolist()
        print("   first bad rows", bad)
