"""A stand-in for the original project's hot-path modules, so that `neuman_b200.install()` can be exercised without the
reference tree.  `standin()` registers `utils.render_utils`, `utils.ray_utils`, `models.vanilla` and `models.human_nerf`
in `sys.modules` with the reference's names and call signatures; install() then rebinds them exactly as it rebinds the
reference's modules.  What a wrapper falls through to -- "the reference's own implementation" -- is the oracle restatement
(oracle/neuman_oracle.py, pinned to the reference's stored outputs by tests/test_oracle_vs_reference.py), and the networks
are neuman_b200's mirror modules with the reference's plain torch forward."""
import contextlib
import sys
import types

from neuman_b200 import models as nbm
from oracle import neuman_oracle as no

NAMES = ("utils", "utils.render_utils", "utils.ray_utils", "models", "models.vanilla", "models.human_nerf")


class Joiner(nbm.Joiner):
    """models/vanilla.py:155-166: the encodings and the network as torch ops (any device, differentiable)."""

    def forward(self, input_pts, input_views=None):
        return self.nerf(self.pos_pe(input_pts), self.dir_pe(input_views))


class OffsetNet(nbm.OffsetNet):
    pass


class HumanNeRF(nbm.HumanNeRF):
    pass


for _c in (Joiner, OffsetNet, HumanNeRF):
    _c.__module__ = "models.human_nerf" if _c is HumanNeRF else "models.vanilla"


def build_nerf(opt):
    coarse, fine = nbm.build_nerf(opt)
    coarse.__class__ = fine.__class__ = Joiner
    return coarse, fine


# ---- utils/render_utils.py ----
def raw2outputs(raw, z_vals, rays_d, raw_noise_std=0, white_bkg=True):
    return no.raw2outputs(raw, z_vals, rays_d, raw_noise_std, white_bkg)


def render_vanilla(coarse_net, cap, fine_net=None, rays_per_batch=32768, samples_per_ray=64, importance_samples_per_ray=128,
                   white_bkg=True, return_depth=False):
    H, W = cap.shape
    rgb, dep = no.render_vanilla(no.net_params_from_joiner(coarse_net),
                                 no.net_params_from_joiner(fine_net) if fine_net is not None else None,
                                 cap.intrinsic_matrix, cap.cam_pose.camera_to_world, H, W, cap.near["bkg"], cap.far["bkg"],
                                 rays_per_batch=rays_per_batch, samples_per_ray=samples_per_ray,
                                 importance_samples_per_ray=importance_samples_per_ray, white_bkg=white_bkg)
    rgb, dep = rgb.reshape(H, W, 3), dep.reshape(H, W)
    return (rgb, dep) if return_depth else rgb


def _cuda_only(name):
    def fn(*a, **k):
        raise NotImplementedError(f"stand-in {name}: only the CUDA path is exercised")
    fn.__name__ = name
    return fn


# ---- utils/ray_utils.py ----
def ray_to_samples(ray_batch, samples_per_ray, lindisp=False, perturb=0., device='cpu', append_t=None):
    assert append_t is None
    return no.ray_to_samples(ray_batch["origin"], ray_batch["direction"], ray_batch["near"], ray_batch["far"],
                             samples_per_ray, lindisp, perturb)


def ray_to_importance_samples(ray_batch, z_vals, weights, importance_samples_per_ray, device='cpu', including_old=True,
                              append_t=None):
    assert append_t is None
    return no.ray_to_importance_samples(ray_batch["origin"], ray_batch["direction"], z_vals, weights,
                                        importance_samples_per_ray, including_old)


def sample_pdf(bins, weights, N_samples, det=False, device='cpu'):
    return no.sample_pdf(bins, weights, N_samples, det)


def geometry_guided_near_far(orig, dir, vert, geo_threshold=0.1):
    return no.geometry_guided_near_far(orig, dir, vert, geo_threshold)


def warp_samples_to_canonical(pts, verts, faces, T):
    return no.warp_samples_to_canonical(pts, verts, faces, T)


@contextlib.contextmanager
def standin():
    """Registers the stand-in modules; on exit puts back whatever install() rebound and unregisters them."""
    saved = {n: sys.modules.get(n) for n in NAMES}
    mods = {n: types.ModuleType(n) for n in NAMES}
    ru, ry, mv, hn = mods["utils.render_utils"], mods["utils.ray_utils"], mods["models.vanilla"], mods["models.human_nerf"]
    ru.raw2outputs, ru.render_vanilla = raw2outputs, render_vanilla
    for n in ("render_smpl_nerf", "render_hybrid_nerf", "render_hybrid_nerf_multi_persons"):
        setattr(ru, n, _cuda_only(n))
    ry.ray_to_samples, ry.ray_to_importance_samples, ry.sample_pdf = ray_to_samples, ray_to_importance_samples, sample_pdf
    ry.geometry_guided_near_far, ry.warp_samples_to_canonical = geometry_guided_near_far, warp_samples_to_canonical
    ry.warp_samples_to_canonical_diff = _cuda_only("warp_samples_to_canonical_diff")
    mv.Joiner, mv.OffsetNet, mv.build_nerf = Joiner, OffsetNet, build_nerf
    hn.HumanNeRF = HumanNeRF
    mods["utils"].render_utils, mods["utils"].ray_utils = ru, ry
    mods["models"].vanilla, mods["models"].human_nerf = mv, hn
    sys.modules.update(mods)
    try:
        yield types.SimpleNamespace(render_utils=ru, ray_utils=ry, vanilla=mv, human_nerf=hn)
    finally:
        from neuman_b200 import dropin
        dropin.uninstall()
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m
