"""Drop-in: rebinds the reference's hot-path functions to the CUDA path (SURVEY.md §8b).

    import neuman_b200; neuman_b200.install("/path/to/ml-neuman")
    # or: python -m neuman_b200.run render_test_views.py --scene_dir ...

After install(), `utils.render_utils.render_vanilla / render_smpl_nerf / render_hybrid_nerf /
render_hybrid_nerf_multi_persons / raw2outputs`, `utils.ray_utils.ray_to_samples /
ray_to_importance_samples / sample_pdf / geometry_guided_near_far / warp_samples_to_canonical` and
`models.vanilla.Joiner.forward` (inference, CUDA tensors, grad disabled) run on
libneuman_b200; the reference's nn.Modules, checkpoints and CLI scripts are untouched.  Calls that need
autograd (training) keep the reference's own torch implementation unless `train=True`.

Every wrapper checks that the call is one the CUDA path implements (device, architecture, encoding options) and
otherwise falls through to the reference's own function, so installing never changes results for unsupported
configurations.  install() is idempotent: the reference's originals are stashed on their modules once and every
call re-wraps from those.
"""
import importlib
import sys

import torch

_ORIG = "_neuman_b200_originals"


def _originals(mod, names):
    """The reference's own attributes of `mod` (stashed at the first install)."""
    store = mod.__dict__.get(_ORIG)          # own attribute only (classes: not an inherited one)
    if store is None:
        store = {}
        setattr(mod, _ORIG, store)
    for n in names:
        if n not in store:
            store[n] = getattr(mod, n)
    return store


def supported_joiner(j):
    """True when `j` is a Joiner the kernels implement: 8x256 trunk, skip after layer 4, no output scaling, 10
    log-spaced position frequencies with the input included, 'posenc' or 'rotate' mapping, and either view directions
    (4 direction frequencies, same conditions) or no view directions with output_linear [4,256] (use_viewdirs=False:
    the direction encoding is never used).  A NeRF-T net (--ablate_nerft: position input (x, y, z, t)) qualifies with
    view directions and the 'posenc' position mapping."""
    try:
        n, pp = j.nerf, j.pos_pe
        if pp.input_dims == 4 and (not n.use_viewdirs or pp.mapping != "posenc"):
            return False
        if not n.use_viewdirs:
            return bool(len(n.pts_linears) == 8 and tuple(n.skips) == (4,)
                        and tuple(n.pts_linears[1].weight.shape) == (256, 256)
                        and tuple(n.output_linear.weight.shape) == (4, 256)
                        and getattr(n, "scale_type", "no") == "no"
                        and pp.N_freqs == 10 and pp.input_dims == 3 and pp.log_sampling and pp.include_input
                        and pp.mapping in ("posenc", "rotate"))
        dp = j.dir_pe
        return bool(n.use_viewdirs and len(n.pts_linears) == 8 and tuple(n.skips) == (4,)
                    and tuple(n.pts_linears[1].weight.shape) == (256, 256)
                    and getattr(n, "scale_type", "no") == "no"
                    and pp.N_freqs == 10 and dp.N_freqs == 4 and pp.input_dims in (3, 4) and dp.input_dims == 3
                    and pp.log_sampling and dp.log_sampling and pp.include_input and dp.include_input
                    and pp.mapping in ("posenc", "rotate") and dp.mapping in ("posenc", "rotate")
                    and float(dp.max_freq) == 3.0 and float(getattr(dp, "min_freq", 0)) == 0.0)
    except AttributeError:
        return False


def install(reference_root=None, train=False):
    """train=True additionally routes the trainers' autograd path to the CUDA training kernels: Joiner.forward of
    8x256 nets (gradients to the parameters and to input_pts / input_views, which is what
    trainers/human_nerf_trainer.py:241-278 differentiates through) and raw2outputs with respect to `raw`
    (trainers/vanilla_nerf_trainer.py:45-96), the human trainer's libigl queries to the device BVH, its differentiable
    warp (`warp_samples_to_canonical_diff`, utils/ray_utils.py:69-93) and `HumanNeRF.vertex_forward`
    (models/human_nerf.py:92-122) to the forward / adjoint kernels of csrc/human_train.cu and csrc/smpl.cu."""
    if reference_root and reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    from . import autograd, ops, render

    def on_cuda(*ts):
        return all(isinstance(t, torch.Tensor) and t.is_cuda for t in ts)

    def on_cuda_nograd(*ts):
        return (not torch.is_grad_enabled()) and on_cuda(*ts)

    ru = importlib.import_module("utils.render_utils")
    ry = importlib.import_module("utils.ray_utils")
    mv = importlib.import_module("models.vanilla")
    o_ru = _originals(ru, ("raw2outputs", "render_vanilla", "render_smpl_nerf", "render_hybrid_nerf",
                           "render_hybrid_nerf_multi_persons"))
    o_ry = _originals(ry, ("ray_to_samples", "ray_to_importance_samples", "sample_pdf", "geometry_guided_near_far",
                           "warp_samples_to_canonical", "warp_samples_to_canonical_diff"))
    o_joiner = _originals(mv.Joiner, ("forward",))

    # ---- networks (models/vanilla.py:155-177) ----
    ref_forward = o_joiner["forward"]

    def joiner_forward(self, input_pts, input_views=None):
        viewless = not getattr(self.nerf, "use_viewdirs", True)
        if ((viewless and on_cuda(input_pts)) or (input_views is not None and on_cuda(input_pts, input_views))) \
                and supported_joiner(self):
            if not torch.is_grad_enabled():
                return ops.joiner_forward(self, input_pts, input_views)
            if train and not (ops.is_nerft(self) and (input_pts.requires_grad or input_views.requires_grad)):
                return autograd.joiner_forward(self, input_pts, input_views)   # (no input gradients for NeRF-T nets)
        return ref_forward(self, input_pts, input_views)          # other training / CPU / other architectures
    mv.Joiner.forward = joiner_forward

    # ---- offset networks (models/vanilla.py:169-177): a Joiner on the tensor-core kernels when the time column is constant ----
    ref_off_forward = _originals(mv.OffsetNet, ("forward",))["forward"]

    def offset_forward(self, input_pts, cur_iter=None):
        if cur_iter is None and on_cuda(input_pts) and (train or not torch.is_grad_enabled()):
            from . import models
            out = models.offset_forward_tc_if_constant_time(self, input_pts)
            if out is not None:
                return out
        return ref_off_forward(self, input_pts, cur_iter)
    mv.OffsetNet.forward = offset_forward

    # ---- composite (utils/render_utils.py:69-105) ----
    ref_raw2outputs = o_ru["raw2outputs"]

    def raw2outputs(raw, z_vals, rays_d, raw_noise_std=0, white_bkg=True):
        if on_cuda_nograd(raw, z_vals, rays_d):
            return ops.raw2outputs(raw, z_vals, rays_d, raw_noise_std, white_bkg)
        if (train and torch.is_grad_enabled() and on_cuda(raw, z_vals, rays_d)
                and not z_vals.requires_grad and not rays_d.requires_grad):
            return autograd.raw2outputs(raw, z_vals, rays_d, raw_noise_std, white_bkg)
        return ref_raw2outputs(raw, z_vals, rays_d, raw_noise_std, white_bkg)
    raw2outputs.__name__ = "raw2outputs"
    ru.raw2outputs = raw2outputs

    # ---- frame drivers (utils/render_utils.py:108-461) ----
    def nets_of(name, model, a, k):
        if name == "render_vanilla":
            fine = k.get("fine_net", a[1] if len(a) > 1 else None)
            return [model] + ([fine] if fine is not None else [])
        if name == "render_smpl_nerf":
            return [model.coarse_human_net]
        if name == "render_hybrid_nerf":
            return [model.coarse_bkg_net, model.fine_bkg_net, model.coarse_human_net]
        humans = k.get("human_models", a[1] if len(a) > 1 else [])
        return [model.coarse_bkg_net, model.fine_bkg_net] + [h.coarse_human_net for h in humans]

    def supported_call(name, model, a, k):
        # render_vanilla(ablate_nerft=True) renders NeRF-T nets at the frame's time; every other call takes plain nets
        nerft = name == "render_vanilla" and bool(k.get("ablate_nerft", False))
        try:
            nets = nets_of(name, model, a, k)
            if not all(next(n.parameters()).is_cuda and supported_joiner(n) and ops.is_nerft(n) == nerft for n in nets):
                return False
            if nerft:
                cap = k.get("cap", a[0] if a else None)
                float(cap.frame_id["frame_id"]) / float(cap.frame_id["total_frames"])
        except (AttributeError, StopIteration, TypeError, KeyError, ZeroDivisionError):
            return False
        return not k.get("ablate_nerft", False) or nerft

    for name in ("render_vanilla", "render_smpl_nerf", "render_hybrid_nerf", "render_hybrid_nerf_multi_persons"):
        ref_fn, new_fn = o_ru[name], getattr(render, name)

        def make(name=name, ref_fn=ref_fn, new_fn=new_fn):
            def wrapped(model, *a, **k):
                if supported_call(name, model, a, k):
                    return new_fn(model, *a, **k)
                return ref_fn(model, *a, **k)
            wrapped.__name__ = ref_fn.__name__
            wrapped.__doc__ = ref_fn.__doc__
            return wrapped
        setattr(ru, name, make())

    # ---- samplers and geometry (utils/ray_utils.py) ----
    ref_rts, ref_rtis, ref_pdf = o_ry["ray_to_samples"], o_ry["ray_to_importance_samples"], o_ry["sample_pdf"]
    ref_gg, ref_warp = o_ry["geometry_guided_near_far"], o_ry["warp_samples_to_canonical"]

    def constants_of_the_step(*ts):
        return on_cuda(*ts) and (not torch.is_grad_enabled() or train)

    def time_ok(append_t):
        # the time column is concatenated as given (:133-134): any tensor that is a constant of the step
        return append_t is None or (isinstance(append_t, torch.Tensor) and not append_t.requires_grad)

    def ray_to_samples(ray_batch, samples_per_ray, lindisp=False, perturb=0., device='cpu', append_t=None):
        if time_ok(append_t) and constants_of_the_step(ray_batch['origin'], ray_batch['near']):
            return ops.ray_to_samples(ray_batch, samples_per_ray, lindisp, perturb, append_t=append_t)
        return ref_rts(ray_batch, samples_per_ray, lindisp, perturb, device, append_t)

    def ray_to_importance_samples(ray_batch, z_vals, weights, importance_samples_per_ray, device='cpu',
                                  including_old=True, append_t=None):
        if time_ok(append_t) and constants_of_the_step(z_vals, weights):       # samples are constants of the step (:150 detaches)
            return ops.ray_to_importance_samples(ray_batch, z_vals, weights, importance_samples_per_ray,
                                                 including_old=including_old, append_t=append_t)
        return ref_rtis(ray_batch, z_vals, weights, importance_samples_per_ray, device, including_old, append_t)

    def sample_pdf(bins, weights, N_samples, det=False, device='cpu'):
        if constants_of_the_step(bins, weights):
            return ops.sample_pdf(bins, weights, N_samples, det)
        return ref_pdf(bins, weights, N_samples, det, device)

    def geometry_guided_near_far(orig, dir, vert, geo_threshold=ops.DEFAULT_GEO_THRESH):
        if on_cuda(orig, dir) and isinstance(vert, torch.Tensor) and not any(t.requires_grad for t in (orig, dir, vert)):
            return ops.geometry_guided_near_far(orig, dir, vert, geo_threshold)
        return ref_gg(orig, dir, vert, geo_threshold)

    def warp_samples_to_canonical(pts, verts, faces, T):
        # the reference takes numpy arrays and returns float64 numpy (utils/ray_utils.py:48-66); CUDA tensors take the
        # device path and come back as CUDA tensors (what its callers build next, utils/render_utils.py:226-227)
        if isinstance(pts, torch.Tensor) and pts.is_cuda:
            return ops.warp_samples_to_canonical(pts, verts, faces, T)
        return ref_warp(pts, verts, faces, T)
    ry.ray_to_samples, ry.ray_to_importance_samples, ry.sample_pdf = ray_to_samples, ray_to_importance_samples, sample_pdf
    ry.geometry_guided_near_far, ry.warp_samples_to_canonical = geometry_guided_near_far, warp_samples_to_canonical

    ref_diff = o_ry["warp_samples_to_canonical_diff"]
    if train:
        # the human trainer's CPU libigl queries (utils/ray_utils.py:70, trainers/human_nerf_trainer.py:310,326)
        def warp_samples_to_canonical_diff(pts, verts, faces, T):
            if isinstance(verts, torch.Tensor) and verts.is_cuda and isinstance(T, torch.Tensor) and T.is_cuda:
                T_inv, f_id, sd = ops.warp_samples_to_canonical_diff(pts, verts, faces, T)
                return T_inv, f_id.cpu().numpy(), sd.cpu().numpy()        # the reference returns igl's numpy arrays
            return ref_diff(pts, verts, faces, T)
        ry.warp_samples_to_canonical_diff = warp_samples_to_canonical_diff
        try:
            igl = importlib.import_module("igl")
            ref_sd = _originals(igl, ("signed_distance",))["signed_distance"]

            def signed_distance(P, V, F, *a, **k):
                if a or k or not torch.cuda.is_available():
                    return ref_sd(P, V, F, *a, **k)
                return ops.signed_distance(P, V, F)
            igl.signed_distance = signed_distance
        except (ImportError, AttributeError):
            pass
    else:
        ry.warp_samples_to_canonical_diff = ref_diff

    # ---- HumanNeRF.vertex_forward (models/human_nerf.py:92-122): the per-step SMPL transforms of the human trainer ----
    hn = importlib.import_module("models.human_nerf")
    ref_vf = _originals(hn.HumanNeRF, ("vertex_forward",))["vertex_forward"]
    if train:
        def vertex_forward(self, idx, pose=None, beta=None):
            bm = getattr(self, "body_model", None)
            try:
                ok = bm is not None and bm.v_template.is_cuda and self.poses.is_cuda and self.da_smpl.is_cuda
            except AttributeError:
                ok = False
            if not ok:
                return ref_vf(self, idx, pose, beta)
            dm = getattr(bm, "_nm_device_model", None)
            if dm is None:
                n_betas = int(self.betas.shape[-1])
                dm = ops.SmplModelDevice(bm.v_template, bm.shapedirs[:, :, :n_betas], bm.J_regressor, bm.lbs_weights, bm.parents,
                                         device=bm.v_template.device)
                bm._nm_device_model = dm
            pose = self.poses[idx][None] if pose is None else pose
            beta = self.betas[idx][None] if beta is None else beta
            return autograd.vertex_forward(dm, pose, beta, self.alignments[idx], float(self.scale), self.da_smpl)
        hn.HumanNeRF.vertex_forward = vertex_forward
    else:
        hn.HumanNeRF.vertex_forward = ref_vf
    return {"render_utils": ru, "ray_utils": ry, "vanilla": mv, "human_nerf": hn}


def uninstall():
    """Puts the reference's own functions back (tests)."""
    for name in ("utils.render_utils", "utils.ray_utils", "models.vanilla", "models.human_nerf", "igl"):
        mod = sys.modules.get(name)
        if mod is None:
            continue
        targets = [mod] + ([mod.Joiner, mod.OffsetNet] if name == "models.vanilla" else []) + ([mod.HumanNeRF] if name == "models.human_nerf" else [])
        for t in targets:
            for k, v in t.__dict__.get(_ORIG, {}).items():
                setattr(t, k, v)
