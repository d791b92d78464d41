"""Frame renderers with the reference's signatures and return conventions
(utils/render_utils.py:108-461): numpy float32 H x W x 3 (and H x W) arrays.  Each one is a single
call into the C ABI frame driver; `rays_per_batch` is accepted for signature compatibility only (it
bounds memory in the reference and does not change results).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib, ops
from ._lib import NmRenderOpts

DEFAULT_GEO_THRESH = ops.DEFAULT_GEO_THRESH
CHUNK = 32768            # device-side rays per chunk
SMPL_CHUNK = 262144      # human-only renders: few rays hit, one hit-count read-back per chunk -> fewer, larger chunks (7 KB / ray)


def _device_of(net):
    return next(net.parameters()).device


def _opts(S, N, white_bkg, near=0.0, far=1.0, geo=DEFAULT_GEO_THRESH, render_can=False, interval_comp=1.0, chunk=CHUNK):
    o = NmRenderOpts()
    o.samples_per_ray, o.importance_samples_per_ray = int(S), int(N)
    o.white_bkg = int(bool(white_bkg))
    o.mlp_mode = ops._mlp_mode()
    o.rays_per_batch = int(chunk)
    o.render_can = int(bool(render_can))
    o.near_bkg, o.far_bkg = float(near), float(far)
    o.geo_threshold, o.interval_comp = float(geo), float(interval_comp)
    return o


def _range_policy(ctx):
    """After a call that already synchronised (host output): fail loudly if a tensor-core MLP launch saturated an fp16
    operand (NM_ERR_RANGE).  NEUMAN_RANGE_POLICY=warn|ignore relaxes it."""
    import os
    import warnings
    pol = os.environ.get("NEUMAN_RANGE_POLICY", "error")
    if pol == "ignore":
        return
    try:
        ctx.range_check()
    except _lib.NmError as e:
        if pol == "warn":
            warnings.warn(str(e), RuntimeWarning)
        else:
            raise


def _pinned(n, cols=None):
    shape = (n,) if cols is None else (n, cols)
    return torch.empty(shape, dtype=torch.float32, pin_memory=True)


def _pixel_args(pixels, cap, pix0, n, device):
    """(n, device pointer or NULL): `pixels` = int32 CUDA tensor of row-major pixel indices (a rank's shard)."""
    H, W = cap.shape
    if pixels is None:
        return (H * W - pix0 if n is None else n), None
    if not (isinstance(pixels, torch.Tensor) and pixels.is_cuda and pixels.dtype == torch.int32 and pixels.is_contiguous()):
        raise TypeError("pixels must be a contiguous int32 CUDA tensor of row-major pixel indices")
    if pixels.device != device:
        raise RuntimeError("pixels must live on the networks' device")
    return int(pixels.numel()), pixels


def _outputs(out, n, host_out, device, with_acc):
    """Caller-provided output tensors (`out` = (rgb [n,3], depth [n][, acc [n]]), e.g. slices of a gather buffer) or fresh."""
    if out is not None:
        for t in out:
            if t is not None and (not t.is_contiguous() or t.dtype != torch.float32 or (t.is_cuda == bool(host_out))):
                raise TypeError("out tensors must be contiguous float32 on the side host_out selects")
        assert out[0].numel() == 3 * n and out[1].numel() == n
        return tuple(out) if (not with_acc or len(out) == 3) else tuple(out) + (torch.empty(n, device=device),)
    if host_out:
        return (_pinned(n, 3), _pinned(n)) + ((_pinned(n),) if with_acc else ())
    return (torch.empty(n, 3, device=device), torch.empty(n, device=device)) + ((torch.empty(n, device=device),) if with_acc else ())


def _render(device, cap, pix0, n, pixels, out, host_out, planes, driver):
    """The part every range renderer shares: resolves the pixel range or list, provides the output tensors (planes = 2:
    rgb, depth; 3: + acc), runs driver(ctx, cam, n, pixels, *outputs) under the device guard and applies the range
    policy after a host-output call.  `driver` holds the driver-specific part (net slots, meshes, options, the ctypes
    call with the pointers it is given) and returns the call's status.  Returns the output tensors."""
    if device.type != "cuda":
        raise RuntimeError("neuman_b200 renderers need the networks on a CUDA device (no CPU fallback)")
    ctx = ops._device_ctx(device)
    n, pix = _pixel_args(pixels, cap, pix0, n, device)
    with torch.cuda.device(device):
        outs = _outputs(out, n, host_out, device, planes == 3)[:planes]
        ctx.check(driver(ctx, ops.camera_struct(cap), n, ops._p(pix), *map(ops._p, outs)))
        if host_out:
            _range_policy(ctx)
    return outs


def render_vanilla_range(coarse_net, cap, fine_net=None, samples_per_ray=64, importance_samples_per_ray=128,
                         white_bkg=True, near_far_source='bkg', pix0=0, n=None, host_out=True, chunk=CHUNK, pixels=None,
                         out=None, frame_time=None):
    """Renders the row-major pixel range [pix0, pix0+n), or the pixel list `pixels` (int32 CUDA tensor). host_out: pinned
    host tensors (device->host copy inside the call) else CUDA tensors. frame_time: NeRF-T nets, the time of every
    sample (nm_render_vanilla_t). Returns (rgb [n,3], depth [n])."""
    def driver(ctx, cam, n, pix, rgb, depth):
        cs = ops.net_slot(coarse_net, ctx)
        fs = ops.net_slot(fine_net, ctx) if fine_net is not None else -1
        o = _opts(samples_per_ray, importance_samples_per_ray if fine_net is not None else 0, white_bkg,
                  cap.near[near_far_source], cap.far[near_far_source], chunk=chunk)
        if frame_time is not None:
            return ctx.lib.nm_render_vanilla_t(ctx.h, cs, fs, C.byref(cam), C.byref(o), float(frame_time), pix0, n, pix, rgb,
                                               depth, int(host_out), ctx.stream())
        return ctx.lib.nm_render_vanilla(ctx.h, cs, fs, C.byref(cam), C.byref(o), pix0, n, pix, rgb, depth, int(host_out),
                                         ctx.stream())
    return _render(_device_of(coarse_net), cap, pix0, n, pixels, out, host_out, 2, driver)


def render_vanilla(coarse_net, cap, fine_net=None, rays_per_batch=32768, samples_per_ray=64,
                   importance_samples_per_ray=128, white_bkg=True, near_far_source='bkg', return_depth=False,
                   ablate_nerft=False):
    """utils/render_utils.py:108-161.  ablate_nerft: NeRF-T nets, rendered at the frame's time frame_id / total_frames
    in float32 (what `torch.ones(...) * cur_time` holds, :135-137)."""
    t = None
    if ablate_nerft:
        t = float(np.float32(cap.frame_id['frame_id'] / cap.frame_id['total_frames']))
    rgb, depth = render_vanilla_range(coarse_net, cap, fine_net, samples_per_ray, importance_samples_per_ray, white_bkg,
                                      near_far_source, frame_time=t)
    H, W = cap.shape
    rgb = rgb.numpy().reshape(H, W, 3)
    if return_depth:
        return rgb, depth.numpy().reshape(H, W)
    return rgb


def render_smpl_nerf_range(net, cap, posed_verts, faces, Ts, samples_per_ray=64, white_bkg=True, render_can=False,
                           geo_threshold=DEFAULT_GEO_THRESH, interval_comp=1.0, pix0=0, n=None, host_out=True,
                           chunk=SMPL_CHUNK, pixels=None, out=None):
    device = _device_of(net)
    if Ts is None:      # canonical rendering never reads T (utils/render_utils.py:214-216)
        Ts = np.tile(np.eye(4)[None], (np.asarray(posed_verts).shape[0], 1, 1))

    def driver(ctx, cam, n, pix, rgb, depth, acc):
        hs = ops.net_slot(net.coarse_human_net, ctx)
        ops.set_mesh(posed_verts, faces, Ts, 0, device)
        o = _opts(samples_per_ray, 0, white_bkg, geo=geo_threshold, render_can=render_can, interval_comp=interval_comp,
                  chunk=chunk)
        return ctx.lib.nm_render_smpl_nerf(ctx.h, hs, 0, C.byref(cam), C.byref(o), pix0, n, pix, rgb, depth, acc,
                                           int(host_out), ctx.stream())
    return _render(device, cap, pix0, n, pixels, out, host_out, 3, driver)


def render_smpl_nerf(net, cap, posed_verts, faces, Ts, rays_per_batch=32768, samples_per_ray=64, white_bkg=True,
                     render_can=False, geo_threshold=DEFAULT_GEO_THRESH, return_depth=False, return_mask=False,
                     interval_comp=1.0):
    """utils/render_utils.py:164-246."""
    rgb, depth, acc = render_smpl_nerf_range(net, cap, posed_verts, faces, Ts, samples_per_ray, white_bkg, render_can,
                                             geo_threshold, interval_comp)
    H, W = cap.shape
    rgb, depth, acc = rgb.numpy().reshape(H, W, 3), depth.numpy().reshape(H, W), acc.numpy().reshape(H, W)
    if return_depth and return_mask:
        return rgb, depth, acc
    if return_depth:
        return rgb, depth
    if return_mask:
        return rgb, acc
    return rgb


def _hybrid(bkg_model, human_models, cap, posed_verts, faces, Ts, S, N, white_bkg, geo, multi, pix0, n, host_out, chunk,
            pixels=None, out=None):
    device = _device_of(bkg_model)

    def driver(ctx, cam, n, pix, rgb, depth, acc):
        cs = ops.net_slot(bkg_model.coarse_bkg_net, ctx)
        fs = ops.net_slot(bkg_model.fine_bkg_net, ctx) if bkg_model.fine_bkg_net is not None else -1
        na = len(human_models)
        hs = (C.c_int32 * na)(*[ops.net_slot(m.coarse_human_net, ctx) for m in human_models])
        ac = (C.c_int32 * na)(*range(na))
        for a in range(na):
            ops.set_mesh(posed_verts[a], faces[a], Ts[a], a, device)
        o = _opts(S, N if fs >= 0 else 0, white_bkg, cap.near['bkg'], cap.far['bkg'], geo=geo, chunk=chunk)
        return ctx.lib.nm_render_hybrid(ctx.h, cs, fs, na, hs, ac, int(multi), C.byref(cam), C.byref(o), pix0, n, pix, rgb,
                                        depth, acc, int(host_out), ctx.stream())
    return _render(device, cap, pix0, n, pixels, out, host_out, 3, driver)


def render_hybrid_nerf_range(net, cap, posed_verts, faces, Ts, samples_per_ray=64, importance_samples_per_ray=128,
                             white_bkg=True, geo_threshold=DEFAULT_GEO_THRESH, pix0=0, n=None, host_out=True,
                             chunk=CHUNK, pixels=None, out=None):
    return _hybrid(net, [net], cap, [posed_verts], [faces], [Ts], samples_per_ray, importance_samples_per_ray, white_bkg,
                   geo_threshold, False, pix0, n, host_out, chunk, pixels=pixels, out=out)


def render_hybrid_nerf(net, cap, posed_verts, faces, Ts, rays_per_batch=32768, samples_per_ray=64,
                       importance_samples_per_ray=128, white_bkg=True, geo_threshold=DEFAULT_GEO_THRESH,
                       return_depth=False):
    """utils/render_utils.py:249-362."""
    rgb, depth, _ = render_hybrid_nerf_range(net, cap, posed_verts, faces, Ts, samples_per_ray,
                                             importance_samples_per_ray, white_bkg, geo_threshold)
    H, W = cap.shape
    if return_depth:
        return rgb.numpy().reshape(H, W, 3), depth.numpy().reshape(H, W)
    return rgb.numpy().reshape(H, W, 3)


def render_hybrid_nerf_multi_persons(bkg_model, cap, human_models, posed_verts, faces, Ts, rays_per_batch=32768,
                                     samples_per_ray=64, importance_samples_per_ray=128, white_bkg=True,
                                     geo_threshold=DEFAULT_GEO_THRESH, return_depth=False, pix0=0, n=None):
    """utils/render_utils.py:365-461."""
    rgb, depth, _ = _hybrid(bkg_model, list(human_models), cap, list(posed_verts), list(faces), list(Ts), samples_per_ray,
                            importance_samples_per_ray, white_bkg, geo_threshold, True, pix0, n, True, CHUNK)
    H, W = cap.shape
    if n is not None:
        return (rgb.numpy(), depth.numpy()) if return_depth else rgb.numpy()
    if return_depth:
        return rgb.numpy().reshape(H, W, 3), depth.numpy().reshape(H, W)
    return rgb.numpy().reshape(H, W, 3)


class SimpleCapture:
    """Minimal stand-in for the reference's capture objects (cameras/captures.py:21): exposes exactly the
    attributes the renderers read -- intrinsic_matrix, cam_pose.camera_to_world, shape/size, near/far."""

    class _Pose:
        def __init__(self, c2w):
            self.camera_to_world = np.asarray(c2w)

        @property
        def camera_center_in_world(self):
            return self.camera_to_world[:3, 3]

    def __init__(self, K, c2w, H, W, near=0.0, far=1.0):
        self.intrinsic_matrix = np.asarray(K, dtype=np.float64)
        self.cam_pose = SimpleCapture._Pose(c2w)
        self.shape = (int(H), int(W))
        self.size = self.shape
        self.near = {'bkg': near}
        self.far = {'bkg': far}
