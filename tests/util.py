import os

import numpy as np
import torch

from oracle import neuman_oracle as no
from oracle import scenes, synth_smpl

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden(name):
    return dict(np.load(os.path.join(GOLD, name)))


def product_nets(device="cpu"):
    """(coarse, fine, human) seeded exactly like tools/make_golden.py."""
    import neuman_b200 as nb
    coarse, fine = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False), 1)
    human, _ = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False, posenc="rotate"), 2)
    return coarse.to(device), fine.to(device), human.to(device)


def product_human_model(device="cpu"):
    import neuman_b200 as nb
    torch.manual_seed(1)
    net = nb.HumanNeRF(nb.default_opt(use_cuda=False))
    scenes.boost_density(net.coarse_human_net)
    return net.to(device)


def oracle_params(joiner):
    return no.net_params_from_joiner(joiner)


# ---------------------------------------------------------------------------------------------
# Torch restatements of the two kernel launches of the Joiner backward (neuman_b200.autograd._chain_kernel and
# _dw_kernel), with the same signatures: a test puts them in place of the kernels and compares the gradients.
# ---------------------------------------------------------------------------------------------
def chain_torch(joiner, P, stash, g):
    """The chain of k_mlp_tc_bwd restated with torch GEMMs on the same stash (same masks, same fp16 rounding
    points): the cross-check of the kernel in tests/test_gpu_train.py."""
    from neuman_b200.autograd import _mm32, _pow2_scale
    sx, sf, sv, sm = stash
    n_pe = joiner.pos_pe.out_dim
    scale = _pow2_scale(g, 256.0)
    inv = 1.0 / scale

    def wh(name):
        return P[name].detach().half()
    gs = g * scale
    g_v = ((gs[:, :3] @ P['rgb_linear.weight'].detach().float()) * (sv > 0)).half()
    g_f = _mm32(g_v, wh('views_linears.0.weight')[:, :256].contiguous()).half()
    dX = _mm32(g_f, wh('feature_linear.weight')) + gs[:, 3:4] * P['alpha_linear.weight'].detach().float()
    g_pre = torch.empty_like(sx)
    for l in range(7, -1, -1):
        g_pre[l] = (dX * (sx[l] > 0)).half()
        if l > 0:
            w = wh('pts_linears.%d.weight' % l)
            dX = _mm32(g_pre[l], w[:, n_pe:].contiguous() if l == 5 else w)
    return g_pre, g_f, g_v, inv


def dw_torch(ctx, g_pre, g_f, g_v, sx, sf, n):
    """k_dw_gemm restated: cuBLAS GEMMs on the fp16 planes with fp32 output, bias gradients as fp32 column sums."""
    from neuman_b200.autograd import _mm32
    dw = torch.zeros(9, 256, 256, device=g_pre.device, dtype=torch.float32)
    db = torch.zeros(9, 256, device=g_pre.device, dtype=torch.float32)
    for k in range(7):
        dw[k] = _mm32(g_pre[k + 1].t(), sx[k])
        db[k] = g_pre[k + 1].float().sum(0)
    dw[7] = _mm32(g_f.t(), sx[7])
    db[7] = g_f.float().sum(0)
    dw[8, :128] = _mm32(g_v.t(), sf)
    db[8, :128] = g_v.float().sum(0)
    return dw, db


def bodies():
    return (synth_smpl.random_body(seed=1, center=(0.1, 0.0, 0.3)),
            synth_smpl.random_body(seed=4, center=(-0.15, 0.0, 0.5)))


def psnr(a, b):
    mse = float(np.mean((np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)) ** 2))
    return 99.0 if mse == 0 else -10.0 * np.log10(mse)


# ---------------------------------------------------------------------------------------------
# Depth / colour gates with the measured 11-bit-operand floor (SURVEY.md §8d "noise floor next to every gate").
# north_star: <= 1e-4 abs against the reference path.  The default MLP mode multiplies fp16 operands (11 significand
# bits, like TF32); `floor16` is what that operand precision alone does to the ORACLE's own result on the same rays.  The
# tensor-core path is held to max(1e-4, K * floor16) with K = 1.5 (accumulation order, MUFU encodings); the fp32
# CUDA-core mode (NEUMAN_MLP_MODE=simt) to 1e-4.
# ---------------------------------------------------------------------------------------------
TOL = 1e-4
K_FLOOR = 1.5


def tc_mode():
    return os.environ.get("NEUMAN_MLP_MODE", "tc") != "simt"


def floors16(run):
    """run() -> tuple of numpy arrays (the oracle on some rays); returns max |fp32 - 11-bit operands| per output."""
    base = run()
    with no.precision(operands="f16"):
        tc = run()
    return [float(np.abs(np.asarray(a) - np.asarray(b)).max()) for a, b in zip(base, tc)]


def gate(err, floor16):
    """The bound for a maximum error `err` given the measured floor (see above)."""
    return max(TOL, K_FLOOR * floor16) if tc_mode() else TOL
