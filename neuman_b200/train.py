"""Training step of the background NeRF on the CUDA path: host mirror of
trainers/vanilla_nerf_trainer.py:45-96 (`loss_func`) and :206-223 (`train_batch`).

Forward = the inference kernels (ray_to_samples, Joiner training kernel, raw2outputs, inverse-CDF
resampling); backward = raw2outputs adjoint kernel + the MLP adjoint chain (neuman_b200/autograd.py).
Sample positions are constants of the step exactly as in the reference (`z_samples.detach()`,
utils/ray_utils.py:186-192), so no gradient crosses the samplers.
"""
import torch
import torch.nn.functional as F

from . import autograd, ops


def vanilla_loss_func(coarse_net, fine_net, batch, opt, penalize_empty_space=0., empty_space_loss_fn=F.l1_loss,
                      t_rand=None, noise=None, check_bad_weights=True):
    """trainers/vanilla_nerf_trainer.py:45-96.  batch: origin/direction [R,3], near/far [R], color [R,3]
    (and depth [R] when penalize_empty_space > 0).  Returns the reference's four losses.
    `t_rand` / `noise` = (coarse, fine) pairs let a test fix the stratified jitter and the density noise.
    `check_bad_weights` keeps the reference's dead-density re-initialisation (:84-89); it costs one host
    sync per step, pass False to run the step fully asynchronously.
    opt.ablate_nerft: NeRF-T nets; every sample carries its ray's time batch['viewf_list'] [R,1] as a fourth position
    column (:47-50)."""
    dev = next(coarse_net.parameters()).device
    coarse_time = fine_time = None
    if getattr(opt, 'ablate_nerft', False):
        tv = batch['viewf_list'].to(dev).reshape(-1, 1)
        coarse_time = tv.repeat(1, opt.samples_per_ray)[..., None]
        fine_time = tv.repeat(1, opt.samples_per_ray + opt.importance_samples_per_ray)[..., None]
    perturb = getattr(opt, 'perturb', 0.)
    noise_std = getattr(opt, 'raw_noise_std', 0.)
    color = batch['color'].to(dev)
    pts, dirs, z_vals = ops.ray_to_samples(batch, opt.samples_per_ray, perturb=perturb, device=dev,
                                           t_rand=t_rand, append_t=coarse_time)
    _b, _n = z_vals.shape
    out = coarse_net(pts, dirs)
    rgb_map, _, _, weights, _ = autograd.raw2outputs(out, z_vals, dirs[:, 0, :], raw_noise_std=noise_std,
                                                     white_bkg=opt.white_bkg, noise=None if noise is None else noise[0])
    coarse_rgb_loss = F.mse_loss(rgb_map, color)
    coarse_empty = torch.zeros_like(coarse_rgb_loss)
    if penalize_empty_space > 0:
        depth = batch['depth'].to(dev)[:, None].repeat(1, _n)
        m = z_vals < (depth * opt.margin)
        s = out[m][:, 3]
        coarse_empty = coarse_empty + empty_space_loss_fn(torch.tanh(torch.relu(s)), torch.zeros_like(s)) * penalize_empty_space
    fine_rgb_loss, fine_empty, F_out = torch.zeros_like(coarse_rgb_loss), torch.zeros_like(coarse_rgb_loss), None
    if fine_net is not None:
        F_pts, F_dirs, F_z = ops.ray_to_importance_samples(batch, z_vals, weights.detach(),
                                                           opt.importance_samples_per_ray, device=dev, append_t=fine_time)
        F_out = fine_net(F_pts, F_dirs)
        F_rgb, _, _, _, _ = autograd.raw2outputs(F_out, F_z, F_dirs[:, 0, :], raw_noise_std=noise_std,
                                                 white_bkg=opt.white_bkg, noise=None if noise is None else noise[1])
        fine_rgb_loss = F.mse_loss(F_rgb, color)
        if penalize_empty_space > 0:
            F_depth = batch['depth'].to(dev)[:, None].repeat(1, F_z.shape[1])
            m = F_z < (F_depth * opt.margin)
            s = F_out[m][:, 3]
            fine_empty = fine_empty + empty_space_loss_fn(torch.tanh(torch.relu(s)), torch.zeros_like(s)) * penalize_empty_space
    if check_bad_weights:
        dead = out.detach()[..., 3].max() <= 0.0
        if F_out is not None:
            dead = dead | (F_out.detach()[..., 3].max() <= 0.0)
        if bool(dead):
            print('bad weights, reinitializing')
            coarse_net.apply(weight_reset)
            if fine_net is not None:
                fine_net.apply(weight_reset)
            zero = torch.tensor(0.0, requires_grad=True).float().to(dev)
            return zero, zero, zero, zero
    return coarse_rgb_loss, coarse_empty, fine_rgb_loss, fine_empty


def weight_reset(m):
    """models/vanilla.py:11-13."""
    if isinstance(m, torch.nn.Linear):
        m.reset_parameters()


def train_batch(coarse_net, fine_net, optimizer, batch, opt, iteration=0, nan_guard='device', **kw):
    """trainers/vanilla_nerf_trainer.py:206-223.  Returns the total loss as a 0-d tensor (no host sync
    unless the caller reads it).

    The reference skips the backward pass when the loss is NaN (:214-218).  Here the backward is an fp16-operand chain
    with one power-of-two loss scale, so an overflow can also show up in the gradients only.  nan_guard:
      'device' (default) -- no host sync: if the loss or any gradient is non-finite the step is skipped on the device:
                            the gradients are zeroed, and the parameters and every optimizer state tensor on their device
                            (Adam's moments) are put back to their values before optimizer.step(), which would otherwise
                            still move them by the momentum.  A step counter the optimizer keeps on the host (torch's
                            non-capturable Adam) still counts the skipped step: reading the flag there is what 'host' does;
      'host'             -- the reference's behaviour: read the loss on the host, zero_grad() and skip backward on NaN;
      None               -- no guard."""
    optimizer.zero_grad()
    c_rgb, c_emp, f_rgb, f_emp = vanilla_loss_func(coarse_net, fine_net, batch, opt, **kw)
    total = c_rgb + f_rgb
    if iteration >= getattr(opt, 'delay_iters', 0):
        total = total + c_emp + f_emp
    if nan_guard == 'host':
        if not bool(torch.isfinite(total.detach())):
            print('loss is nan during training')
            optimizer.zero_grad()
        else:
            total.backward()
        optimizer.step()
        return total.detach()
    total.backward()
    if nan_guard == 'device':
        params = [p for g in optimizer.param_groups for p in g['params'] if p.grad is not None]
        if params:
            grads = [p.grad for p in params]
            ok = torch.isfinite(total.detach()) & torch.isfinite(torch.stack(torch._foreach_norm(grads))).all()
            for g in grads:
                g.masked_fill_(~ok, 0.0)
            dev = params[0].device
            kept = [p.data for p in params] + [t for p in params for t in optimizer.state.get(p, {}).values()
                                               if isinstance(t, torch.Tensor) and t.device == dev and t.is_floating_point()]
            saved = torch._foreach_mul(kept, 1.0)
            optimizer.step()
            # kept = kept * ok + saved * (1 - ok): exact for either value of the flag (the step ran on zero gradients,
            # so nothing in kept is non-finite unless it already was)
            okf = ok.float()
            torch._foreach_mul_(kept, okf)
            torch._foreach_mul_(saved, 1.0 - okf)
            torch._foreach_add_(kept, saved)
            return total.detach()
    optimizer.step()
    return total.detach()


def eval_human_samples(net, batch, opt, faces, offset_net=None, t_rand=None, actor=ops.NM_MAX_ACTORS - 1):
    """HumanNeRFTrainer._eval_human_samples (trainers/human_nerf_trainer.py:241-278) on the CUDA path.

    net: neuman_b200.HumanNeRF built with per-frame SMPL parameters and a body model; batch: a HumanRayBatcher /
    HumanRayDataset batch (origin, direction, human_near, human_far, cur_view_f, cap_id); faces: the SMPL faces [F,3]
    (the reference reads them from the capture's posed mesh, :268); offset_net: one of net.offset_nets (the reference draws
    `random.choice(self.net.offset_nets)`, :261) or None to skip the offset.

    Stages: ray_to_samples kernel (:248-257) -> offset network (:260-261; the step's time is one number, so the network
    runs as a Joiner on the tensor-core kernels, models.OffsetNet) -> vertex_forward
    training kernels (:264) -> closest-face query on the device BVH + fused blend / inverse / apply / offset / directions
    (:265-276, nm_signed_distance + nm_human_canonicalize) -> canonical human network on the tensor-core training kernel
    (:277).  loss.backward() then runs the adjoint kernels of every stage: gradients reach the human network, the offset
    network, and net.poses / net.betas / net.alignments.
    Returns the reference's tuple (human_pts [R*S,3], human_dirs, human_z_vals, can_pts, can_dirs, human_out)."""
    dev = next(net.coarse_human_net.parameters()).device
    human_batch = {'origin': batch['origin'].to(dev), 'direction': batch['direction'].to(dev),
                   'near': batch['human_near'].to(dev), 'far': batch['human_far'].to(dev)}
    human_pts, human_dirs, human_z_vals = ops.ray_to_samples(human_batch, opt.samples_per_ray, perturb=getattr(opt, 'perturb', 0.),
                                                             device=dev, t_rand=t_rand)
    human_b, human_n, _ = human_pts.shape
    offset = None
    if offset_net is not None:
        from . import models
        if human_pts.is_cuda and models.offset_tc_supported(offset_net):
            offset = models.offset_forward_at_time(offset_net, human_pts, float(batch['cur_view_f']))   # tensor-core kernels
        else:
            cur_time = torch.ones_like(human_pts[..., 0:1]) * float(batch['cur_view_f'])
            offset = offset_net(torch.cat([human_pts, cur_time], dim=-1))
    mesh, raw_Ts = net.vertex_forward(int(batch['cap_id']))
    can_pts, can_dirs, _, _ = ops.eval_human_samples(human_pts, mesh[0], faces, raw_Ts[0], offset=offset, actor=actor)
    human_out = net.coarse_human_net(can_pts, can_dirs)
    return human_pts.reshape(-1, 3), human_dirs, human_z_vals, can_pts, can_dirs, human_out
