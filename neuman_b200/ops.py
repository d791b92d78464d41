"""CUDA-backed stage functions with the reference's names, argument meaning and return conventions
(utils/ray_utils.py, utils/render_utils.py, models/vanilla.py).  Tensors must live on a CUDA
device; every function fails loudly otherwise -- there is no CPU path in this package.
"""
import ctypes as C
import itertools
import os
import weakref

import numpy as np
import torch

from . import _lib
from ._lib import Context, NmCamera, NmNerfDesc, NmNerfNoviewDesc, NM_MAX_ACTORS

DEFAULT_GEO_THRESH = 0.2     # utils/constant.py:14


def _mlp_mode():
    return _lib.NM_MLP_SIMT_F32 if os.environ.get("NEUMAN_MLP_MODE", "tc") == "simt" else _lib.NM_MLP_TC_F16


def _device_ctx(device):
    """The library context of a CUDA torch.device; a device without an index is the current one."""
    return Context.get(device.index if device.index is not None else torch.cuda.current_device())


def _ctx_for(t):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("neuman_b200 ops need CUDA tensors (no CPU fallback)")
    return _device_ctx(t.device)


def _f32(t, device=None):
    if not isinstance(t, torch.Tensor):
        t = torch.as_tensor(np.asarray(t))
    if device is not None and t.device != device:
        t = t.to(device)
    return t.contiguous().float()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


# ---------------------------------------------------------------------------------------------
# networks
# ---------------------------------------------------------------------------------------------
_PE_KIND = {"posenc": _lib.NM_PE_POSENC, "rotate": _lib.NM_PE_ROTATE}


_uid_counter = itertools.count(1)


def _net_uid(joiner):
    """Process-unique id of a Joiner, assigned at its first pack.  (id() is reused by CPython after garbage collection,
    and the caching allocator hands a new net the same storage with _version 0: an id()-based key then matches
    the dead net's slot.)"""
    tag = joiner.__dict__.get("_nm_uid")
    if tag is None or tag[1] != id(joiner):         # never packed, or a copy.deepcopy that inherited the attribute
        tag = (next(_uid_counter), id(joiner))
        joiner.__dict__["_nm_uid"] = tag
    return tag[0]


def _net_key(joiner):
    # (data_ptr, _version) per parameter detects in-place updates and `.data = ...` swaps to other storage
    return (_net_uid(joiner),) + tuple((p.data_ptr(), p._version) for p in joiner.nerf.parameters())


def _evict_uid(ctx_ref, uid):
    ctx = ctx_ref()
    if ctx is None:
        return
    for k in [k for k in ctx.slots if k[0] == uid]:
        ctx.slot_keys[ctx.slots.pop(k)] = None


def invalidate_net(joiner):
    """Forget the packed copy of `joiner` on every device (call after replacing parameter storage in a way that
    keeps data_ptr and _version, e.g. `p.data.copy_()` through a non-tracking view)."""
    tag = joiner.__dict__.get("_nm_uid")
    if tag is not None:
        for ctx in list(Context._by_device.values()):
            _evict_uid(weakref.ref(ctx), tag[0])


def is_viewless(joiner):
    """True for a view-independent net (NeRF with use_viewdirs=False: one output_linear head, no direction input)."""
    return not getattr(joiner.nerf, "use_viewdirs", True)


def is_nerft(joiner):
    """True for a NeRF-T net (the reference's --ablate_nerft background nets): its position input is (x, y, z, t)."""
    return int(getattr(joiner.pos_pe, "input_dims", 3)) == 4


def net_slot(joiner, ctx=None):
    """Packs (lazily, keyed on a per-module uid + parameter storage + version) a Joiner into a library slot: a
    view-dependent net (use_viewdirs=True) with nm_net_pack, a view-independent one (use_viewdirs=False, output_linear
    [4,256]) with nm_net_pack_noview, a NeRF-T net (4-D posenc position input, view-dependent) with nm_net_pack_nerft."""
    nerf = joiner.nerf
    viewless, nerft = is_viewless(joiner), is_nerft(joiner)
    if nerft and (viewless or joiner.pos_pe.mapping != "posenc"):
        raise NotImplementedError("NeRF-T nets: only view-dependent nets with the posenc position mapping are built")
    p0 = nerf.pts_linears[0].weight
    ctx = ctx or _ctx_for(p0)
    key = _net_key(joiner)
    if key in ctx.slots:
        s = ctx.slots[key]
        ctx.slot_clock += 1
        ctx.slot_used[s] = ctx.slot_clock
        return s
    if viewless and tuple(nerf.output_linear.weight.shape) != (4, 256):
        raise NotImplementedError("view-independent nets: only output_linear [4,256] (output_ch=4) is built")
    if viewless and getattr(nerf, "scale_type", "no") != "no":
        raise NotImplementedError("view-independent nets: only scale_type='no' is built")
    if len(nerf.pts_linears) != 8 or nerf.pts_linears[1].weight.shape != (256, 256) or tuple(nerf.skips) != (4,):
        raise NotImplementedError("only the 8x256, skips=[4] architecture is built (reference default)")
    # stale entries of the same module
    uid = key[0]
    _evict_uid(weakref.ref(ctx), uid)
    if uid not in ctx.finalized_uids:                                # release the slot when the module is garbage-collected
        ctx.finalized_uids.add(uid)
        weakref.finalize(joiner, _evict_uid, weakref.ref(ctx), uid)
    free = [i for i, k in enumerate(ctx.slot_keys) if k is None]
    if free:
        s = free[0]
    else:
        s = int(np.argmin(ctx.slot_used))
        ctx.slots.pop(ctx.slot_keys[s], None)
    d = NmNerfNoviewDesc() if viewless else NmNerfDesc()
    keep = []

    def dev(t):
        c = t.detach().contiguous().float()
        if c.data_ptr() != t.data_ptr():
            keep.append(c)                          # a converted temporary: must outlive the pack kernels
        return c.data_ptr()
    for i in range(8):
        d.pts_w[i] = dev(nerf.pts_linears[i].weight)
        d.pts_b[i] = dev(nerf.pts_linears[i].bias)
    pp = joiner.pos_pe
    d.pos_pe_kind = _PE_KIND[pp.mapping]
    d.pos_min_freq, d.pos_max_freq, d.pos_n_freqs = float(pp.min_freq), float(pp.max_freq), int(pp.N_freqs)
    if viewless:
        d.output_w, d.output_b = dev(nerf.output_linear.weight), dev(nerf.output_linear.bias)
        ctx.check(ctx.lib.nm_net_pack_noview(ctx.h, s, C.byref(d), ctx.stream()))
    else:
        d.feature_w, d.feature_b = dev(nerf.feature_linear.weight), dev(nerf.feature_linear.bias)
        d.alpha_w, d.alpha_b = dev(nerf.alpha_linear.weight), dev(nerf.alpha_linear.bias)
        d.views_w, d.views_b = dev(nerf.views_linears[0].weight), dev(nerf.views_linears[0].bias)
        d.rgb_w, d.rgb_b = dev(nerf.rgb_linear.weight), dev(nerf.rgb_linear.bias)
        dp = joiner.dir_pe
        d.dir_pe_kind = _PE_KIND[dp.mapping]
        d.dir_min_freq, d.dir_max_freq, d.dir_n_freqs = float(dp.min_freq), float(dp.max_freq), int(dp.N_freqs)
        pack = ctx.lib.nm_net_pack_nerft if nerft else ctx.lib.nm_net_pack
        ctx.check(pack(ctx.h, s, C.byref(d), ctx.stream()))
    if keep:
        torch.cuda.current_stream(ctx.device).synchronize()  # `keep` temporaries may be freed after this
    ctx.slots[key] = s
    ctx.slot_keys[s] = key
    ctx.slot_clock += 1
    ctx.slot_used[s] = ctx.slot_clock
    return s


def joiner_forward(joiner, input_pts, input_views=None, mode=None):
    """Joiner.forward (models/vanilla.py:162-166) -> [...,4].  A view-independent net ignores input_views (may be None),
    as the reference does (:145-146); a NeRF-T net takes input_pts [...,4] = (x, y, z, t)."""
    viewless = is_viewless(joiner)
    if input_views is None and not viewless:
        raise NotImplementedError("use_viewdirs=True networks need input_views")
    ctx = _ctx_for(input_pts)
    slot = net_slot(joiner, ctx)
    shape = input_pts.shape[:-1]
    pts = _f32(input_pts).reshape(-1, 4 if is_nerft(joiner) else 3)
    views = None
    if not viewless:
        views = _f32(input_views, pts.device).reshape(-1, 3)
        assert views.shape[0] == pts.shape[0], "input_views must match input_pts"
    raw = torch.empty(pts.shape[0], 4, device=pts.device, dtype=torch.float32)
    ctx.check(ctx.lib.nm_mlp_forward(ctx.h, slot, _mlp_mode() if mode is None else mode, _p(pts), _p(views),
                                     pts.shape[0], 0, _p(raw), ctx.stream()))
    return raw.reshape(*shape, 4)


def mlp_forward_rays(joiner, origins, dirs, z_vals, mode=None):
    """Fused `ray_to_samples` point generation + Joiner.forward: pts = o + d*z, views = d."""
    ctx = _ctx_for(z_vals)
    slot = net_slot(joiner, ctx)
    o, d, z = _f32(origins, z_vals.device), _f32(dirs, z_vals.device), _f32(z_vals)
    R, S = z.shape
    raw = torch.empty(R, S, 4, device=z.device, dtype=torch.float32)
    ctx.check(ctx.lib.nm_mlp_forward_rays(ctx.h, slot, _mlp_mode() if mode is None else mode, _p(o), _p(d), _p(z), R, S,
                                          _p(raw), ctx.stream()))
    return raw


# ---------------------------------------------------------------------------------------------
# rays / sampling
# ---------------------------------------------------------------------------------------------
def camera_struct(cap):
    """cap: any object with .intrinsic_matrix (3x3), .cam_pose.camera_to_world (4x4), .shape (H,W)."""
    cam = NmCamera()
    K = np.asarray(cap.intrinsic_matrix, dtype=np.float64).reshape(-1)
    c2w = np.asarray(cap.cam_pose.camera_to_world, dtype=np.float64).reshape(-1)
    for i in range(9):
        cam.K[i] = K[i]
    for i in range(16):
        cam.c2w[i] = c2w[i]
    cam.H, cam.W = int(cap.shape[0]), int(cap.shape[1])
    return cam


def shot_rays(cap, xys, device=None):
    """utils/ray_utils.py:23-29 -> (origins, dirs) float32 CUDA tensors [n,3]."""
    device = torch.device(device or "cuda")
    ctx = _device_ctx(device)
    if isinstance(xys, torch.Tensor) and xys.is_cuda:           # already on the device (neuman_b200/data.py)
        device = xys.device
        ctx = _device_ctx(device)
        xy = xys[:, :2].to(torch.int32).contiguous()
    else:
        xy = torch.as_tensor(np.ascontiguousarray(np.asarray(xys)[:, :2]).astype(np.int32)).to(device)
    n = xy.shape[0]
    o = torch.empty(n, 3, device=device)
    d = torch.empty(n, 3, device=device)
    cam = camera_struct(cap)
    with torch.cuda.device(device):
        ctx.check(ctx.lib.nm_raygen(ctx.h, C.byref(cam), 0, 0, n, _p(xy), _p(o), _p(d), ctx.stream()))
    return o, d


def shot_all_rays(cap, device=None, mode=1):
    """utils/ray_utils.py:32-38 (+ the .float() of render_utils.py:114-115)."""
    device = torch.device(device or "cuda")
    ctx = _device_ctx(device)
    n = int(cap.shape[0]) * int(cap.shape[1])
    o = torch.empty(n, 3, device=device)
    d = torch.empty(n, 3, device=device)
    cam = camera_struct(cap)
    with torch.cuda.device(device):
        ctx.check(ctx.lib.nm_raygen(ctx.h, C.byref(cam), mode, 0, n, None, _p(o), _p(d), ctx.stream()))
    return o, d


def geometry_guided_near_far(orig, dir, vert, geo_threshold=DEFAULT_GEO_THRESH):
    """utils/ray_utils.py:197-233 (CUDA tensors in, CUDA tensors out)."""
    ctx = _ctx_for(orig)
    o, d = _f32(orig), _f32(dir, orig.device)
    v = _f32(vert, o.device)
    near = torch.empty(o.shape[0], device=o.device)
    far = torch.empty(o.shape[0], device=o.device)
    ctx.check(ctx.lib.nm_near_far(ctx.h, _p(o), _p(d), o.shape[0], _p(v), v.shape[0], float(geo_threshold),
                                  _p(near), _p(far), ctx.stream()))
    return near, far


def near_far_mesh(orig, dir, actor, geo_threshold=DEFAULT_GEO_THRESH):
    """geometry_guided_near_far against the mesh of `actor` (set_mesh), computed as the frame drivers do."""
    ctx = _ctx_for(orig)
    o, d = _f32(orig), _f32(dir, orig.device)
    near = torch.empty(o.shape[0], device=o.device)
    far = torch.empty(o.shape[0], device=o.device)
    with torch.cuda.device(o.device):
        ctx.check(ctx.lib.nm_near_far_mesh(ctx.h, int(actor), _p(o), _p(d), o.shape[0], float(geo_threshold),
                                           _p(near), _p(far), ctx.stream()))
    return near, far


def ray_to_samples(ray_batch, samples_per_ray, lindisp=False, perturb=0., device='cuda', append_t=None, t_rand=None):
    """utils/ray_utils.py:96-135 -> (pts [R,S,3], dirs [R,S,3], z_vals [R,S]); with append_t [R,S,1] the time column is
    concatenated to pts ([R,S,4]) as the reference does (:133-134)."""
    o = _f32(ray_batch['origin'])
    ctx = _ctx_for(o)
    d = _f32(ray_batch['direction'], o.device)
    near = _f32(ray_batch['near'], o.device).reshape(-1)
    far = _f32(ray_batch['far'], o.device).reshape(-1)
    R = o.shape[0]
    assert near.shape[0] == far.shape[0] == R
    S = int(samples_per_ray)
    pts = torch.empty(R, S, 3, device=o.device)
    dirs = torch.empty(R, S, 3, device=o.device)
    z = torch.empty(R, S, device=o.device)
    tr = None
    if perturb > 0.:
        tr = _f32(t_rand, o.device) if t_rand is not None else torch.rand(R, S, device=o.device)
    ctx.check(ctx.lib.nm_ray_to_samples(ctx.h, _p(o), _p(d), _p(near), _p(far), 0.0, 0.0, R, S, int(bool(lindisp)),
                                        _p(tr), _p(pts), _p(dirs), _p(z), ctx.stream()))
    if append_t is not None:
        pts = torch.cat([pts, append_t.to(pts.device)], dim=-1)
    return pts, dirs, z


def sample_pdf(bins, weights, N_samples, det=False, device='cuda', u=None):
    """utils/ray_utils.py:164-194."""
    b = _f32(bins)
    ctx = _ctx_for(b)
    w = _f32(weights, b.device)
    R, B = b.shape
    assert w.shape == (R, B - 1)
    if u is None and not det:
        u = torch.rand(R, N_samples, device=b.device)
    uu = _f32(u, b.device) if u is not None else None
    out = torch.empty(R, N_samples, device=b.device)
    ctx.check(ctx.lib.nm_sample_pdf(ctx.h, _p(b), _p(w), R, B, int(N_samples), _p(uu), _p(out), ctx.stream()))
    return out


def ray_to_importance_samples(ray_batch, z_vals, weights, importance_samples_per_ray, device='cuda',
                              including_old=True, append_t=None):
    """utils/ray_utils.py:138-160 (append_t: as ray_to_samples, :158-159)."""
    z = _f32(z_vals)
    ctx = _ctx_for(z)
    o, d = _f32(ray_batch['origin'], z.device), _f32(ray_batch['direction'], z.device)
    w = _f32(weights, z.device)
    R, S = z.shape
    N = int(importance_samples_per_ray)
    total = S + N if including_old else N
    pts = torch.empty(R, total, 3, device=z.device)
    dirs = torch.empty(R, total, 3, device=z.device)
    zo = torch.empty(R, total, device=z.device)
    ctx.check(ctx.lib.nm_importance_samples(ctx.h, _p(o), _p(d), _p(z), _p(w), R, S, N, int(bool(including_old)),
                                            _p(pts), _p(dirs), _p(zo), ctx.stream()))
    if append_t is not None:
        pts = torch.cat([pts, append_t.to(pts.device)], dim=-1)
    return pts, dirs, zo


def raw2outputs(raw, z_vals, rays_d, raw_noise_std=0, white_bkg=True, noise=None, sigma_scale=1.0):
    """utils/render_utils.py:69-105 -> (rgb_map, disp_map, acc_map, weights, depth_map)."""
    r = _f32(raw)
    ctx = _ctx_for(r)
    z, d = _f32(z_vals, r.device), _f32(rays_d, r.device)
    R, S = z.shape
    assert r.shape == (R, S, 4) and d.shape == (R, 3)
    nz = None
    if raw_noise_std > 0.:
        nz = _f32(noise, r.device) if noise is not None else torch.randn(R, S, device=r.device) * raw_noise_std
    rgb = torch.empty(R, 3, device=r.device)
    disp, acc, depth = (torch.empty(R, device=r.device) for _ in range(3))
    w = torch.empty(R, S, device=r.device)
    ctx.check(ctx.lib.nm_raw2outputs(ctx.h, _p(r), _p(z), _p(d), R, S, _p(nz), float(sigma_scale), int(bool(white_bkg)),
                                     _p(rgb), _p(disp), _p(acc), _p(w), _p(depth), ctx.stream()))
    return rgb, disp, acc, w, depth


def merge_samples(z_list, raw_list):
    """sort(cat(z)) + gather of raw (utils/render_utils.py:330-337) -> (z_sorted, raw_sorted)."""
    z_list = [_f32(z) for z in z_list]
    ctx = _ctx_for(z_list[0])
    raw_list = [_f32(r, z_list[0].device) for r in raw_list]
    n = len(z_list)
    R = z_list[0].shape[0]
    S = [int(z.shape[1]) for z in z_list]
    zp = (C.c_void_p * n)(*[z.data_ptr() for z in z_list])
    rp = (C.c_void_p * n)(*[r.data_ptr() for r in raw_list])
    sp = (C.c_int32 * n)(*S)
    zo = torch.empty(R, sum(S), device=z_list[0].device)
    ro = torch.empty(R, sum(S), 4, device=z_list[0].device)
    ctx.check(ctx.lib.nm_merge_samples(ctx.h, n, zp, rp, sp, R, _p(zo), _p(ro), ctx.stream()))
    return zo, ro


# ---------------------------------------------------------------------------------------------
# observation -> canonical warp
# ---------------------------------------------------------------------------------------------
_FACES_CACHE = {}


def faces_device(faces, device):
    """faces [F,>=3] (numpy / tensor) -> contiguous int32 [F,3] on `device`.  The topology is the same array step after step
    (the SMPL faces): host arrays are uploaded once and found again by (address, shape, checksum)."""
    device = torch.device(device)
    if isinstance(faces, torch.Tensor):
        if faces.device == device and faces.dtype == torch.int32 and faces.shape[1] == 3 and faces.is_contiguous():
            return faces
        return faces.detach()[:, :3].to(device=device, dtype=torch.int32).contiguous()
    a = np.asarray(faces)
    key = (a.__array_interface__['data'][0], a.shape, a.dtype.str, int(a[:, :3].sum()), str(device))
    hit = _FACES_CACHE.get(key)
    if hit is None:
        if len(_FACES_CACHE) >= 8:
            _FACES_CACHE.pop(next(iter(_FACES_CACHE)))
        hit = torch.from_numpy(np.ascontiguousarray(a[:, :3], dtype=np.int32)).to(device)
        _FACES_CACHE[key] = hit
    return hit


def set_mesh(verts, faces, T, actor=0, device=None):
    """Uploads one actor's per-frame mesh (verts [V,3], faces [F,>=3], T [>=V,4,4] or None) and builds the BVH.
    CUDA tensors are taken from device memory, anything else goes through host arrays."""
    if isinstance(verts, torch.Tensor) and verts.is_cuda:
        device = verts.device
        ctx = _device_ctx(device)
        v = verts.detach().float().contiguous()
        f = faces_device(faces, device)
        t = None
        if T is not None:
            t = (T.detach() if isinstance(T, torch.Tensor) else torch.as_tensor(np.asarray(T))).to(device=device, dtype=torch.float64)
            t = t.contiguous().reshape(-1, 16)
        with torch.cuda.device(device):
            ctx.check(ctx.lib.nm_mesh_set(ctx.h, int(actor), _p(v), v.shape[0], _p(f), f.shape[0], _p(t),
                                          0 if t is None else t.shape[0], 1, ctx.stream()))
        return ctx
    device = torch.device(device or "cuda")
    ctx = _device_ctx(device)
    v = np.ascontiguousarray(verts.detach().cpu().numpy() if isinstance(verts, torch.Tensor) else verts, dtype=np.float32)
    f = np.ascontiguousarray(np.asarray(faces)[:, :3], dtype=np.int32)
    tp, tn = None, 0
    if T is not None:
        t = np.ascontiguousarray(T.detach().cpu().numpy() if isinstance(T, torch.Tensor) else T, dtype=np.float64)
        t = t.reshape(-1, 16)
        tp, tn = t.ctypes.data_as(C.c_void_p), t.shape[0]
    with torch.cuda.device(device):
        ctx.check(ctx.lib.nm_mesh_set(ctx.h, int(actor), v.ctypes.data_as(C.c_void_p), v.shape[0],
                                      f.ctypes.data_as(C.c_void_p), f.shape[0], tp, tn, 0, ctx.stream()))
    return ctx


def signed_distance(pts, verts, faces, actor=NM_MAX_ACTORS - 1, device=None):
    """igl.signed_distance(P, V, F) as the reference calls it (utils/ray_utils.py:70,
    trainers/human_nerf_trainer.py:310,326): (S [n] signed distance, negative inside; I [n] closest face;
    C [n,3] closest point).  numpy in -> float64 / int32 numpy out (igl's types); CUDA tensors in -> CUDA tensors out
    (float64, int32, float64).  Uses the last actor slot by default so that the renderers' meshes stay set."""
    as_numpy = not isinstance(pts, torch.Tensor)
    if isinstance(verts, torch.Tensor) and verts.is_cuda:
        device = verts.device
    device = torch.device(device or (pts.device if isinstance(pts, torch.Tensor) and pts.is_cuda else "cuda"))
    if isinstance(verts, torch.Tensor) and not verts.is_cuda:
        verts = verts.detach().to(device)
    ctx = set_mesh(verts, faces, None, actor, device)
    p = _f32(pts, device).reshape(-1, 3)
    n = p.shape[0]
    S = torch.empty(n, device=p.device, dtype=torch.float64)
    I = torch.empty(n, device=p.device, dtype=torch.int32)
    Cl = torch.empty(n, 3, device=p.device, dtype=torch.float64)
    with torch.cuda.device(p.device):
        ctx.check(ctx.lib.nm_signed_distance(ctx.h, int(actor), _p(p), n, _p(S), _p(I), _p(Cl), ctx.stream()))
    if as_numpy:
        return S.cpu().numpy(), I.cpu().numpy(), Cl.cpu().numpy()
    return S, I, Cl


def warp_samples_to_canonical_diff(pts, verts, faces, T, actor=NM_MAX_ACTORS - 1):
    """utils/ray_utils.py:69-93: the closest-face query (igl.signed_distance on the CPU in the reference, :70) runs on
    the device BVH; the differentiable part -- barycentric coordinates of the closest point from cross products (:72-88),
    blend of the three per-vertex transforms and its inverse (:90-91) -- is one kernel (nm_warp_diff_forward) whose
    adjoint (nm_warp_diff_backward) sends gradients to `verts` and `T` as torch autograd does in the reference.
    pts: [n,3] numpy or tensor (treated as constants); verts [V,3], T [V,4,4]: CUDA tensors.
    Returns (T_interp_inv [n,4,4], f_id [n], signed_dist [n])."""
    from . import autograd
    signed_dist, f_id, closest = signed_distance(torch.as_tensor(np.asarray(pts)) if not isinstance(pts, torch.Tensor) else pts.detach(),
                                                 verts, faces, actor=actor, device=verts.device)
    return autograd.warp_diff_tinv(verts, T, f_id, closest, faces), f_id, signed_dist


def eval_human_samples(pts, verts, faces, T, offset=None, actor=NM_MAX_ACTORS - 1):
    """The geometric part of HumanNeRFTrainer._eval_human_samples (trainers/human_nerf_trainer.py:263-276): samples
    pts [R,S,3] of the observation space -> canonical points (inverse blended transform, + offset) and canonical
    directions, fused (nm_human_canonicalize) and differentiable with respect to verts [V,3], T [V,4,4] and offset [R,S,3].
    Returns (can_pts, can_dirs, f_id [R*S], signed_dist [R*S])."""
    from . import autograd
    p = _f32(pts, verts.device)
    signed_dist, f_id, closest = signed_distance(p.detach().reshape(-1, 3), verts, faces, actor=actor, device=verts.device)
    cp, cd = autograd.human_canonicalize(p, verts, T, f_id, closest, faces, offset)
    return cp, cd, f_id, signed_dist


def warp_samples_to_canonical(pts, verts, faces, T, actor=0, return_face_id=False):
    """utils/ray_utils.py:48-66: pts [R,S,3] -> (can_pts, can_dirs, closest) float32 CUDA tensors (the
    reference returns float64 numpy which its callers immediately cast with .float())."""
    assert len(pts.shape) == 3 and pts.shape[-1] == 3, 'pts should have shape [num_rays, num_samples, 3]'
    if not isinstance(pts, torch.Tensor):
        pts = torch.as_tensor(np.asarray(pts)).cuda()
    p = _f32(pts)
    ctx = set_mesh(verts, faces, T, actor, p.device)
    R, S, _ = p.shape
    cp, cd, cl = (torch.empty(R, S, 3, device=p.device) for _ in range(3))
    fid = torch.empty(R, S, device=p.device, dtype=torch.int32)
    ctx.check(ctx.lib.nm_warp_to_canonical(ctx.h, int(actor), _p(p), R, S, _p(cp), _p(cd), _p(cl), _p(fid), ctx.stream()))
    if return_face_id:
        return cp, cd, cl, fid
    return cp, cd, cl


# ---------------------------------------------------------------------------------------------
# SMPL per-vertex transforms (models/smpl.py, data_io/neuman_helper.py:299-330)
# ---------------------------------------------------------------------------------------------
class SmplModelDevice:
    """Device copy of the SMPL arrays the path reads (models/smpl.py:73-107): v_template [V,3],
    shapedirs [V,3,NB], J_regressor [J,V], weights [V,J], parents [J] (parents[0] = -1)."""

    def __init__(self, v_template, shapedirs, J_regressor, weights, parents, device="cuda"):
        dev = torch.device(device)
        self.v_template = _f32(v_template, dev)
        self.shapedirs = _f32(shapedirs, dev)
        self.J_regressor = _f32(J_regressor, dev)
        self.weights = _f32(weights, dev)
        par = np.asarray(parents.cpu() if isinstance(parents, torch.Tensor) else parents).astype(np.int32).copy()
        par[0] = -1
        self._par = (C.c_int32 * len(par))(*par.tolist())
        self.n_verts, self.n_joints = int(self.v_template.shape[0]), int(len(par))
        self.n_betas = int(self.shapedirs.shape[-1])
        self.device = dev
        m = _lib.NmSmplModel()
        m.v_template, m.shapedirs = self.v_template.data_ptr(), self.shapedirs.data_ptr()
        m.J_regressor, m.weights = self.J_regressor.data_ptr(), self.weights.data_ptr()
        m.parents = self._par
        m.n_verts, m.n_joints, m.n_betas = self.n_verts, self.n_joints, self.n_betas
        self.struct = m


def smpl_verts_transformations(model, poses, betas, concat_joints=False):
    """SMPL.verts_transformations (models/smpl.py:109-162) -> (vertices [V(+J),3], T [V(+J),4,4]) float32 CUDA."""
    ctx = _device_ctx(model.device)
    pose = _f32(poses, model.device).reshape(-1)
    beta = _f32(betas, model.device).reshape(-1)
    n = model.n_verts + (model.n_joints if concat_joints else 0)
    T = torch.empty(n, 4, 4, device=model.device)
    verts = torch.empty(n, 3, device=model.device)
    with torch.cuda.device(model.device):
        ctx.check(ctx.lib.nm_smpl_vertex_transforms(ctx.h, C.byref(model.struct), _p(pose), _p(beta), int(bool(concat_joints)),
                                                    _p(T), _p(verts), ctx.stream()))
    return verts, T


def smpl_scene_transforms(model, pose, betas, alignment, scale):
    """data_io/neuman_helper.py:299-330: returns (world_verts [V,3] f32, world_joints [J,3] f32,
    T_da2scene [V+J,4,4] f64) on the device."""
    ctx = _device_ctx(model.device)
    p = _f32(pose, model.device).reshape(-1)
    da = torch.zeros(model.n_joints, 3, device=model.device)
    da[1, 2], da[2, 2] = 1.0, -1.0                                  # the 'da' pose (:293-297)
    da = da.reshape(-1).contiguous()
    b = _f32(betas, model.device).reshape(-1)
    al = np.ascontiguousarray(np.asarray(alignment, dtype=np.float64).reshape(16))
    alc = (C.c_double * 16)(*al.tolist())
    n = model.n_verts + model.n_joints
    T = torch.empty(n, 4, 4, device=model.device, dtype=torch.float64)
    world = torch.empty(n, 3, device=model.device)
    with torch.cuda.device(model.device):
        ctx.check(ctx.lib.nm_smpl_scene_transforms(ctx.h, C.byref(model.struct), _p(p), _p(da), _p(b), alc, float(scale),
                                                   _p(T), _p(world), ctx.stream()))
    return world[:model.n_verts], world[model.n_verts:], T


def near_far_cache(cap, verts, geo_threshold=DEFAULT_GEO_THRESH, device=None):
    """The per-frame array `export_near_far_cache` writes (data_io/cache_helper.py:16-36): [H,W,3] float64 =
    (near, far, 1) of geometry_guided_near_far for every pixel (inf / -inf where the ray misses).  One ray
    generation + one near/far launch for the whole frame instead of the reference's chunked torch loop."""
    device = torch.device(device or "cuda")
    o, d = shot_all_rays(cap, device=device, mode=0)          # shot_rays semantics over all pixels (:28-29)
    near, far = geometry_guided_near_far(o, d, _f32(verts, device), geo_threshold)
    H, W = int(cap.shape[0]), int(cap.shape[1])
    out = np.ones([H, W, 3])
    out[..., 0] = near.cpu().numpy().reshape(H, W)
    out[..., 1] = far.cpu().numpy().reshape(H, W)
    return out
