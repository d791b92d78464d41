"""neuman_b200 -- H100-native (sm_90a) implementation of NeuMan's ray-marching hot path behind the
reference's own function / module signatures.  See DESIGN.md and INTEGRATION.md.

    import neuman_b200 as nb
    rgb = nb.render_vanilla(coarse, cap, fine_net=fine, samples_per_ray=128, importance_samples_per_ray=128)
    nb.install()     # rebind the reference's utils.render_utils / utils.ray_utils / models.vanilla
"""
from . import _lib
from .models import (Embedder, NeRF, Joiner, OffsetNet, HumanNeRF, SMPL, build_nerf, build_offset_net,      # noqa: F401
                     default_opt)
from .ops import (raw2outputs, ray_to_samples, ray_to_importance_samples, sample_pdf,          # noqa: F401
                  geometry_guided_near_far, warp_samples_to_canonical, warp_samples_to_canonical_diff, signed_distance,
                  shot_rays, shot_all_rays,
                  joiner_forward, mlp_forward_rays, merge_samples, set_mesh)
from .render import (render_vanilla, render_smpl_nerf, render_hybrid_nerf,                     # noqa: F401
                     render_hybrid_nerf_multi_persons, SimpleCapture)
from .dropin import install                                                                   # noqa: F401

__all__ = [n for n in dir() if not n.startswith("_")]
