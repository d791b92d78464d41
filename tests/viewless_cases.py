"""The seeded view-independent cases (use_viewdirs=False nets) shared by tools/make_golden_viewless.py, which renders them
with the unmodified reference, and by tests/test_viewless.py / tests/test_gpu_viewless.py, which hold the oracle and the
kernels to those goldens; plus the exact-window rule of the view-independent output head."""
import numpy as np
import torch

from tests import tc_exact as tx

VAN = dict(H=20, W=28, S=48, N=40)          # the frames.npz vanilla case: camera van_K / van_c2w
HUM = dict(H=22, W=18, S=24, N=16)          # the frames.npz human cases: camera h_K / h_c2w
NET_SEEDS = {"posenc": 3, "rotate": 4}
# human models: (use_viewdirs of the background nets, specular_can = use_viewdirs of the canonical human net, seed)
HUMANS = {"A": (True, False, 1), "B": (False, True, 2)}


def boost_viewless(joiner, gain=8.0, bias=0.3):
    """The view-independent counterpart of synthetic.boost_density: default init leaves sigma ~ +-0.1, so the density
    column of output_linear is scaled and shifted (identically for reference and product nets)."""
    with torch.no_grad():
        joiner.nerf.output_linear.weight[3].mul_(gain)
        joiner.nerf.output_linear.bias[3].add_(bias)
    return joiner


def viewless_nets(build_nerf, default_opt, posenc):
    """(coarse, fine) view-independent Joiners, seeded; build_nerf / default_opt from the reference or from neuman_b200."""
    torch.manual_seed(NET_SEEDS[posenc])
    coarse, fine = build_nerf(default_opt(use_cuda=False, use_viewdirs=False, posenc=posenc))
    return boost_viewless(coarse), boost_viewless(fine)


def human_model(human_nerf_cls, default_opt, which):
    """HumanNeRF with background nets of one kind and a canonical human net of the other (HUMANS[which])."""
    bkg_view, human_view, seed = HUMANS[which]
    torch.manual_seed(seed)
    net = human_nerf_cls(default_opt(use_cuda=False, num_offset_nets=0, use_viewdirs=bkg_view, specular_can=human_view))
    for j in (net.coarse_bkg_net, net.fine_bkg_net, net.coarse_human_net):
        if not j.nerf.use_viewdirs:
            boost_viewless(j)
        elif j is net.coarse_human_net:
            with torch.no_grad():                                    # synthetic.boost_density
                j.nerf.alpha_linear.weight.mul_(8.0)
                j.nerf.alpha_linear.bias.add_(0.3)
    return net


def checksum(module):
    return float(sum(p.detach().double().abs().sum() for p in module.parameters()))


def head_check(W16, W32, sx7, raw):
    """The output head of a view-independent net: raw = the fp32 accumulator of fp16(X7) @ fp16(W_out)^T (K = 256 in
    16-channel MMAs), then one fp32 add of the fp32 output_linear.bias (DESIGN.md §3)."""
    e, B = tx.mma_ref([(sx7, W16['output_linear.weight'])])
    e = e + W32['output_linear.bias']
    return tx.check32("output", raw, e, B + tx.EPS32 * (e.abs() + B))


def outliers(a, ref, tol):
    """Fraction of rays (rows of the [rays, channels] arrays a, ref) with any channel off by more than `tol`."""
    a, ref = np.asarray(a, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    n = ref.shape[0]
    err = np.abs(a.reshape(n, -1) - ref.reshape(n, -1)).max(-1)
    return float((err > tol).mean())


def backward_checks(W16, scale, d_raw, sx, g_pre):
    """Yields a Check for g_pre[7..0] of nm_mlp_backward on a view-independent net, each on the kernel's own inputs:
    g_pre[7] = r16(mask_7 (S g @ W_out)), four fp32 FMAs with fp32 weights in any order (bound 4 u sum|terms|), then the
    hidden layers' K = 256 MMAs from the kernel's own plane above (as tests/tc_exact.py backward_checks)."""
    gs = float(scale) * d_raw.double()
    W32 = W16['_out32']
    e, S = tx.affine(gs, W32.T)
    yield tx.check16("g_pre7", g_pre[7], e, 4 * tx.EPS32 * S, mask=sx[7] > 0)
    npe = tx.n_pos(W16)
    for l in range(7, 0, -1):
        w = W16[f'pts_linears.{l}.weight']
        if l == 5:
            w = w[:, npe:]
        e, B = tx.mma_ref([(g_pre[l], w.T)])
        yield tx.check16(f"g_pre{l - 1}", g_pre[l - 1], e, B, mask=sx[l - 1] > 0)
