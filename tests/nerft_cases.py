"""The seeded NeRF-T cases (the reference's --ablate_nerft background nets: position input (x, y, z, t)) shared by
tools/make_golden_nerft.py, which evaluates and renders them with the unmodified reference, and by tests/test_nerft.py /
tests/test_gpu_nerft.py, which hold the oracle and the kernels to those goldens."""
import numpy as np
import torch

from oracle import neuman_oracle as no

VAN = dict(H=20, W=28, S=48, N=40)          # the frames.npz vanilla case: camera van_K / van_c2w
NET_SEED = 5
FRAMES = ((7, 30), (23, 30))               # (frame_id, total_frames) of the two renders
NEAR, FAR = 0.0, 3.14
T_PAIR = (0.1, 0.9)                        # the same 50 points at two times


def nerft_nets(build_nerf, default_opt):
    """(coarse, fine) NeRF-T Joiners, seeded; build_nerf / default_opt from the reference or from neuman_b200.  The alpha
    head is boosted as synthetic.boost_density does, so that the renders are not degenerate."""
    torch.manual_seed(NET_SEED)
    coarse, fine = build_nerf(default_opt(use_cuda=False, raw_pos_dim=4))
    for j in (coarse, fine):
        with torch.no_grad():
            j.nerf.alpha_linear.weight.mul_(8.0)
            j.nerf.alpha_linear.bias.add_(0.3)
    return coarse, fine


def net_inputs(stages):
    """(pts [400,4], views [400,3]) float32: the 300 stage samples of stages.npz with times 0, 1, k/30 and uniform random
    values (75 rows each), then the first 50 of them at T_PAIR[0] and at T_PAIR[1]."""
    p, v = stages["n_pts"].astype(np.float32), stages["n_views"].astype(np.float32)
    rng = np.random.default_rng(11)
    t = np.concatenate([np.zeros(75), np.ones(75), np.arange(75) % 31 / 30.0, rng.uniform(0, 1, 75)]).astype(np.float32)
    pts = np.concatenate([np.concatenate([p, t[:, None]], 1)] +
                         [np.concatenate([p[:50], np.full((50, 1), tt, np.float32)], 1) for tt in T_PAIR])
    views = np.concatenate([v, v[:50], v[:50]])
    return pts, views


def frame_time(frame_id, total_frames):
    """The time of every sample of a render: `torch.ones(...) * (frame_id / total_frames)` holds float32 of the quotient."""
    return float(np.float32(frame_id / total_frames))


def oracle_render(coarse, fine, K, c2w, H, W, t, S=VAN["S"], N=VAN["N"], white_bkg=True):
    """render_vanilla(..., ablate_nerft=True) (utils/render_utils.py:108-161) from the oracle's stages: the samplers'
    points with a time column of value t (:134-148, utils/ray_utils.py:133-134,158-159), in the oracle's precision.
    Returns (rgb [n,3], depth [n]) float32 numpy."""
    o_all, d_all = no.shot_all_rays(K, c2w, H, W)
    dt = torch.get_default_dtype()
    with torch.no_grad():
        o, d = torch.from_numpy(o_all).to(dt), torch.from_numpy(d_all).to(dt)
        n = o.shape[0]
        pts, dirs, z = no.ray_to_samples(o, d, torch.full((n, 1), NEAR), torch.full((n, 1), FAR), S)
        pts = torch.cat([pts, torch.full(pts.shape[:-1] + (1,), t, dtype=dt)], -1)
        rgb, _, _, w, depth = no.raw2outputs(no.net_forward(coarse, pts, dirs), z, d, white_bkg=white_bkg)
        if fine is not None:
            pts, dirs, z = no.ray_to_importance_samples(o, d, z, w, N)
            pts = torch.cat([pts, torch.full(pts.shape[:-1] + (1,), t, dtype=dt)], -1)
            rgb, _, _, _, depth = no.raw2outputs(no.net_forward(fine, pts, dirs), z, d, white_bkg=white_bkg)
    return rgb.float().numpy(), depth.float().numpy()


# ---- the tensor-core kernel's layer-0 / layer-5 operands of a NeRF-T net, in its K order (csrc/mlp_tc.cu) ----------
def kernel_pos_columns():
    """Columns of the [n,96] encoding plane (nm_encode_f16: the reference's order, 1.0 at 84) that feed the kernel's
    position block channels 0..63: x, y, z, then per frequency sin(x, y, z), cos(x, y, z), then the constant 1."""
    cols = [0, 1, 2]
    for k in range(10):
        cols += [4 + 8 * k + d for d in range(3)] + [8 + 8 * k + d for d in range(3)]
    return cols + [84]


def kernel_time_columns():
    """Columns of the [n,96] plane that feed channels 32..63 of the direction block (the time slab's K slices 2..3):
    t, then sin(f_k t), cos(f_k t) per frequency; 85 (a zero column of the plane) for the channels no input feeds."""
    cols = [3]
    for k in range(10):
        cols += [7 + 8 * k, 11 + 8 * k]
    return cols + [85] * 11


def nerft_blocks(W16, l, pe96, sx, time_cols=None, time_slab=True):
    """(operand, weight) blocks of pts_linears.l (l = 0 or 5) of a NeRF-T net in the order k_mlp_tc_nerft issues them:
    the position block (bias in the column of its channel 63), the activation blocks of layer 5, then the time slab.
    time_cols / time_slab let a test plant a defect in the model's picture of the kernel."""
    w, b = W16[f'pts_linears.{l}.weight'], W16[f'pts_linears.{l}.bias']
    pc = kernel_pos_columns()
    tc = kernel_time_columns() if time_cols is None else time_cols
    wpos = torch.cat([w[:, pc[:63]], b[:, None]], 1)
    wt = torch.zeros(w.shape[0], 32, dtype=w.dtype, device=w.device)
    for j, c in enumerate(tc):
        if c < 84:
            wt[:, j] = w[:, c]
    blocks = [(pe96[:, pc], wpos)]
    if l == 5:
        blocks.append((sx[4], w[:, 84:]))
    if time_slab:
        blocks.append((pe96[:, kernel_time_columns()], wt))
    return blocks


def outliers(a, ref, tol):
    """Fraction of rays (rows of the [rays, channels] arrays a, ref) with any channel off by more than `tol`."""
    a, ref = np.asarray(a, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    n = ref.shape[0]
    err = np.abs(a.reshape(n, -1) - ref.reshape(n, -1)).max(-1)
    return float((err > tol).mean())
