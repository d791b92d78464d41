"""Timing of the human trainer's per-step geometry on one GPU (SURVEY.md §8f-1), reference defaults: 2048 rays x 128 samples
(options/options.py:76-77).  Stages of HumanNeRFTrainer._eval_human_samples (trainers/human_nerf_trainer.py:241-278) and their
adjoints on the CUDA path, next to the same algebra written with torch ops on the same GPU (what the reference's code costs
once its tensors are on the device; its libigl query stays on the CPU and is not timed here).

    python tools/human_train_bench.py > human_train_bench.json
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import neuman_b200 as nb                                   # noqa: E402
from neuman_b200 import autograd as nag, ops, train as nt  # noqa: E402
from neuman_b200.synthetic import make_model               # noqa: E402


def timed(fn, warm=3, reps=10):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def torch_warp_diff(closest, f_id, verts, fa, T):
    """utils/ray_utils.py:72-91 with torch ops (the reference's own algebra, tensors on the device)."""
    tri = verts[fa[f_id.long()]]
    c = closest.float()
    a, b, cc = tri[:, 0], tri[:, 1], tri[:, 2]
    N = torch.cross(b - a, cc - a, dim=-1)
    den = (N * N).sum(-1)
    u = (N * torch.cross(cc - b, c - b, dim=-1)).sum(-1) / den
    v = (N * torch.cross(a - cc, c - cc, dim=-1)).sum(-1) / den
    bary = torch.stack([u, v, 1 - u - v], 1)
    return torch.inverse((T[fa[f_id.long()]] * bary[..., None, None]).sum(1))


def main():
    dev = "cuda"
    out = {"rays": 2048, "samples": 128}
    R, S = 2048, 128
    rng = np.random.RandomState(0)
    nj = 24
    pose = rng.normal(0, 0.3, (1, 3 * nj)).astype(np.float32)
    betas = rng.normal(0, 1.0, (1, 10)).astype(np.float32)
    align = np.eye(4, dtype=np.float32)
    align[3, :3] = (0.3, -0.1, 2.0)
    opt = nb.default_opt(use_cuda=True, num_offset_nets=1, offset_scale=0.02, offset_scale_type='tanh', samples_per_ray=S)
    torch.manual_seed(0)
    net = nb.HumanNeRF(opt, poses=pose, betas=betas, alignments=align[None], scale=0.4, smpl_model=make_model(0))
    F = np.ascontiguousarray(make_model(0)["f"][:, :3].astype(np.int64))
    with torch.no_grad():
        V0 = net.vertex_forward(0)[0][0]
    eye = V0.mean(0) + torch.tensor([0.0, 0.0, -2.0], device=dev)
    tgt = V0[torch.randint(0, V0.shape[0], (R,), device=dev)] + 0.02 * torch.randn(R, 3, device=dev)
    d = tgt - eye
    dist = d.norm(dim=1, keepdim=True)
    batch = {'origin': eye[None].repeat(R, 1), 'direction': d / dist, 'human_near': dist - 0.2, 'human_far': dist + 0.2,
             'cur_view_f': 3 / 11, 'cap_id': 0}
    params = [p for p in net.parameters() if p.requires_grad]

    def step(offset_net):
        for p in params:
            p.grad = None
        o = nt.eval_human_samples(net, batch, opt, F, offset_net=offset_net)
        o[5].square().mean().backward()
    out["step_ms_with_offset_net"] = timed(lambda: step(net.offset_nets[0]))
    out["step_ms_without_offset_net"] = timed(lambda: step(None))
    # ---- stage by stage ----
    pts, dirs, z = ops.ray_to_samples({'origin': batch['origin'], 'direction': batch['direction'], 'near': batch['human_near'],
                                       'far': batch['human_far']}, S)
    m = net.body_model.dev_model
    p_, b_, a_ = net.poses[0][None], net.betas[0][None], net.alignments[0]

    def vf():
        w, T = nag.vertex_forward(m, p_, b_, a_, 0.4, net.da_smpl)
        (w.sum() + T.sum()).backward()
    out["vertex_forward_fwd_bwd_ms"] = timed(vf)
    out["vertex_forward_fwd_ms"] = timed(lambda: nag.vertex_forward(m, p_.detach(), b_.detach(), a_.detach(), 0.4, net.da_smpl))
    with torch.enable_grad():
        mesh, Ts = net.vertex_forward(0)
    verts, T = mesh[0].detach(), Ts[0].detach()
    out["signed_distance_query_ms"] = timed(lambda: nb.signed_distance(pts.reshape(-1, 3), verts, F))
    sd, f_id, closest = nb.signed_distance(pts.reshape(-1, 3), verts, F)
    vg, Tg = verts.clone().requires_grad_(True), T.clone().requires_grad_(True)
    off = (0.01 * torch.randn(R, S, 3, device=dev)).requires_grad_(True)
    out["canonicalize_fwd_ms"] = timed(lambda: nag.human_canonicalize(pts, verts, T, f_id, closest, F, off.detach()))

    def can_fb():
        vg.grad = Tg.grad = off.grad = None
        cp, cd = nag.human_canonicalize(pts, vg, Tg, f_id, closest, F, off)
        (cp.sum() + cd.sum()).backward()
    out["canonicalize_fwd_bwd_ms"] = timed(can_fb)
    fa = torch.from_numpy(F).to(dev)

    def torch_fb():
        vg.grad = Tg.grad = off.grad = None
        Ti = torch_warp_diff(closest, f_id, vg, fa, Tg)
        ph = torch.cat([pts.reshape(-1, 3), torch.ones(R * S, 1, device=dev)], -1)
        cp = (Ti @ ph[..., None])[:, :3, 0].reshape(R, S, 3) + off
        cd = cp[:, 1:] - cp[:, :-1]
        cd = torch.cat([cd, cd[:, -1:]], 1)
        cd = cd / torch.norm(cd, dim=2, keepdim=True)
        (cp.sum() + cd.sum()).backward()
    out["canonicalize_torch_ops_fwd_bwd_ms"] = timed(torch_fb, warm=2, reps=5)
    on = net.offset_nets[0]

    def off_fb():
        for p in on.parameters():
            p.grad = None
        on.forward_library(torch.cat([pts, torch.ones_like(pts[..., :1]) * 0.3], -1)).sum().backward()
    out["offset_net_library_fwd_bwd_ms"] = timed(off_fb, warm=2, reps=5)

    def off_tc():
        for p in on.parameters():
            p.grad = None
        on.forward_at_time(pts, 0.3).sum().backward()
    out["offset_net_tensor_core_fwd_bwd_ms"] = timed(off_tc)
    cp, cd = nag.human_canonicalize(pts, verts, T, f_id, closest, F, None)

    def net_fb():
        for p in net.coarse_human_net.parameters():
            p.grad = None
        net.coarse_human_net(cp.detach().requires_grad_(True), cd.detach().requires_grad_(True)).square().mean().backward()
    out["human_net_fwd_bwd_ms"] = timed(net_fb)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
