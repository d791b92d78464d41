"""torch.autograd bindings of the hand-written backward kernels (SURVEY.md §8f-1: the training-time callers
trainers/vanilla_nerf_trainer.py:45-96, trainers/human_nerf_trainer.py:382-446).  Forward = the same CUDA
kernels as inference; backward = their CUDA adjoints.  CUDA tensors only."""
import ctypes as C

import torch

from . import ops
from .ops import _ctx_for, _f32, _p


class _Raw2Outputs(torch.autograd.Function):
    @staticmethod
    def forward(fctx, raw, z_vals, rays_d, noise, sigma_scale, white_bkg):
        r, z, d = _f32(raw), _f32(z_vals, raw.device), _f32(rays_d, raw.device)
        nz = _f32(noise, raw.device) if noise is not None else None
        outs = ops.raw2outputs(r, z, d, raw_noise_std=1.0 if nz is not None else 0, white_bkg=white_bkg, noise=nz,
                               sigma_scale=sigma_scale)
        fctx.save_for_backward(r, z, d, nz if nz is not None else torch.empty(0, device=r.device))
        fctx.has_noise = nz is not None
        fctx.sigma_scale, fctx.white_bkg = float(sigma_scale), bool(white_bkg)
        fctx.mark_non_differentiable(outs[1])           # disp_map
        return outs

    @staticmethod
    def backward(fctx, g_rgb, g_disp, g_acc, g_w, g_depth):
        r, z, d, nz = fctx.saved_tensors
        ctx = _ctx_for(r)
        R, S = z.shape
        grad_raw = torch.empty_like(r)

        def opt(g):
            return _f32(g, r.device) if g is not None else None
        g_rgb, g_acc, g_w, g_depth = opt(g_rgb), opt(g_acc), opt(g_w), opt(g_depth)
        ctx.check(ctx.lib.nm_raw2outputs_backward(ctx.h, _p(r), _p(z), _p(d), R, S, _p(nz if fctx.has_noise else None),
                                                  fctx.sigma_scale, int(fctx.white_bkg), _p(g_rgb), _p(g_depth), _p(g_acc),
                                                  _p(g_w), _p(grad_raw), ctx.stream()))
        return grad_raw, None, None, None, None, None


def raw2outputs(raw, z_vals, rays_d, raw_noise_std=0, white_bkg=True, noise=None, sigma_scale=1.0):
    """Differentiable raw2outputs (utils/render_utils.py:69-105): gradients flow to `raw` through rgb_map,
    acc_map, weights and depth_map."""
    if raw_noise_std > 0. and noise is None:
        noise = torch.randn(raw.shape[:-1], device=raw.device) * raw_noise_std
    return _Raw2Outputs.apply(raw, z_vals, rays_d, noise if raw_noise_std > 0. else None, sigma_scale, white_bkg)


# ---------------------------------------------------------------------------------------------
# Joiner (positional encodings + 8x256 MLP) under autograd
# ---------------------------------------------------------------------------------------------
def _pow2_scale(t, target):
    """0-d fp32 tensor S = 2^k with max|t| * S in [target/2, target]; no host sync."""
    amax = t.abs().amax().clamp_min(1e-30)
    return torch.exp2(torch.floor(torch.log2(target / amax))).float().reshape(1)


def _mm32(a, b):
    return torch.mm(a, b, out_dtype=torch.float32)


def _bmm32(a, b):
    return torch.bmm(a, b, out_dtype=torch.float32)


_K_CHUNK = 4096         # rows per batch of the K = n weight-gradient GEMMs (_wgrad)


def _wgrad(G, X):
    """G^T @ X over the n rows of G [n, M] and X [n, N] (fp16, row-major) -> fp32 [M, N]: a K = n weight-gradient GEMM.
    One torch.mm with K = n leaves it to cuBLAS to split K, and for some shapes (n ~ 14 000 - 40 000 with 64- or 96-wide
    X on an H100) the kernel it picks reduces the split below fp32: up to 1.5 times the error bound of any fp32
    summation order (tests/dw_exact.py gemm_window_any_order; DESIGN.md §2).  So K is split here: a batched GEMM over
    whole _K_CHUNK-row blocks, which fills the GPU without a split of its own, the fp32 sum of its partials, and the
    remaining rows as one GEMM with K < _K_CHUNK."""
    n = G.shape[0]
    nb = n // _K_CHUNK
    k = nb * _K_CHUNK
    out = None
    if nb:
        out = _bmm32(G[:k].view(nb, _K_CHUNK, G.shape[1]).transpose(1, 2), X[:k].view(nb, _K_CHUNK, X.shape[1])).sum(0)
    if n > k:
        t = _mm32(G[k:].t(), X[k:])
        out = t if out is None else out + t
    return out


class _JoinerMLP(torch.autograd.Function):
    """forward: k_mlp_tc<.., kTrain> (csrc/mlp_tc.cu) = the inference kernel + an fp16 stash of every layer
    output and the ReLU sign words.
    backward: k_mlp_tc_bwd (csrc/mlp_tc_bwd.cu) runs the adjoint chain of NeRF.forward (models/vanilla.py:120-152)
    on the tensor cores and writes S * dL/d(pre-activation) of every layer in fp16 (S = power-of-two loss scale
    chosen from max|dL/d raw| on the device); the weight and bias gradients are the K = n GEMMs  g_l^T @ input_l
    over the stash: k_dw_gemm (csrc/dw_gemm.cu) for the nine 256-wide ones, cuBLAS (torch.mm, fp16 operands / fp32
    accumulate) for the narrow ones against the encodings (k_encode_f16) and dL/d raw.
    Gradients go to the network parameters and, when they require grad, to the sample positions / directions
    (dL/d encoding by two small cuBLAS GEMMs on the gradient planes, then k_pe_backward), which is what the human
    trainer's differentiable warp and offset nets consume (trainers/human_nerf_trainer.py:241-278).
    The two kernel launches sit behind module-level functions (_chain_kernel, _dw_kernel), so that a test can put a
    torch restatement of the same chain in their place (tests/util.py).

    The gradient is the exact adjoint of the fp16-operand forward: ReLU masks are those of the fp16 activations,
    so it differs from an fp32 forward's gradient where a pre-activation changes sign under the rounding
    (DESIGN.md "Training numerics")."""

    @staticmethod
    def forward(fctx, pts, views, joiner, *params):
        ctx = _ctx_for(pts)
        slot = ops.net_slot(joiner, ctx)
        n = pts.shape[0]
        dev = pts.device
        h = dict(device=dev, dtype=torch.float16)
        viewless = ops.is_viewless(joiner)                             # (NeRF-T nets: view-dependent, pts [n,4])
        sx = torch.empty(8, n, 256, **h)
        sf = sv = None                                                 # view-independent nets: no feature / views layer
        if not viewless:
            sf, sv = torch.empty(n, 256, **h), torch.empty(n, 128, **h)
        sm = torch.empty(8 if viewless else 9, n, 8, device=dev, dtype=torch.int32)   # planes 0..7: pts_linears, 8: views layer
        raw = torch.empty(n, 4, device=dev, dtype=torch.float32)
        if n:
            ctx.check(ctx.lib.nm_mlp_forward_train(ctx.h, slot, _p(pts), _p(views), n, 0, _p(raw), _p(sx), _p(sf), _p(sv),
                                                   _p(sm), ctx.stream()))
        fctx.joiner = joiner
        fctx.stash = (sx, sf, sv, sm)
        fctx.param_versions = tuple(p._version for _, p in joiner.nerf.named_parameters())
        fctx.save_for_backward(pts, views, *params)
        return raw

    @staticmethod
    def backward(fctx, g_raw):
        stash = fctx.stash
        fctx.stash = None                     # ~5.5 KB per sample: released as soon as this node has run
        if stash is None:
            raise RuntimeError("this network's activation stash was already consumed by an earlier backward pass "
                               "(backward(retain_graph=True) twice through the same forward): run the forward again")
        joiner = fctx.joiner
        names = [k for k, _ in joiner.nerf.named_parameters()]
        pts, views = fctx.saved_tensors[:2]
        P = dict(zip(names, fctx.saved_tensors[2:]))
        # `params` may be tensors COMPUTED for a carrier module (models.offset_forward_at_time) rather than the module's own
        # parameters: if the carrier was re-loaded since this forward, put the values of this forward back before the chain
        mod_params = [p for _, p in joiner.nerf.named_parameters()]
        if (any(p._version != v for p, v in zip(mod_params, fctx.param_versions))
                and any(P[k] is not p for k, p in zip(names, mod_params))):
            with torch.no_grad():
                for k, p in zip(names, mod_params):
                    p.copy_(P[k])
        g = g_raw.reshape(-1, 4).float().contiguous()
        need_w = any(fctx.needs_input_grad[3:])
        d_pts = d_views = None
        viewless = ops.is_viewless(joiner)
        if g.shape[0] == 0:
            grads = {k: torch.zeros_like(v) for k, v in P.items()}
            d_pts = torch.zeros_like(pts)
            d_views = torch.zeros_like(views) if views is not None and not viewless else None
        else:
            g_pre, g_f, g_v, inv = _chain_kernel(joiner, P, stash, g)
            grads = _weight_grads(joiner, stash, pts, views, g, g_pre, g_f, g_v, inv) if need_w else {}
            if fctx.needs_input_grad[0]:
                d_pts = _input_grad(joiner, P, pts, 0, ((g_pre[0], 'pts_linears.0.weight', 0), (g_pre[5], 'pts_linears.5.weight', 0)), inv)
            if fctx.needs_input_grad[1] and not viewless:       # the views never reach the output of a view-independent net
                d_views = _input_grad(joiner, P, views, 1, ((g_v, 'views_linears.0.weight', 256),), inv)
        out = [grads[k].reshape(P[k].shape).to(P[k].dtype) if fctx.needs_input_grad[3 + i] else None
               for i, k in enumerate(names)]
        return (d_pts, d_views, None, *out)


def _input_grad(joiner, P, x, which, terms, inv):
    """dL/d(pts) or dL/d(views): dL/d(encoding) = sum over the layers that read it of g_l @ W_l[:, encoding columns]
    (cuBLAS, fp16 operands, fp32 out), then the adjoint of Embedder.forward (k_pe_backward)."""
    ctx = _ctx_for(x)
    slot = ops.net_slot(joiner, ctx)
    width = (joiner.pos_pe if which == 0 else joiner.dir_pe).out_dim
    ld = (width + 31) // 32 * 32
    d_enc = None
    for gl, name, col0 in terms:
        w = torch.zeros(gl.shape[1], ld, device=x.device, dtype=torch.float16)
        w[:, :width] = P[name].detach()[:, col0:col0 + width]
        t = _mm32(gl, w)
        d_enc = t if d_enc is None else d_enc + t
    n = x.shape[0]
    d_x = torch.empty(n, 3, device=x.device, dtype=torch.float32)
    ctx.check(ctx.lib.nm_pe_backward(ctx.h, slot, which, _p(x), 0, _p(d_enc), ld, _p(inv.contiguous()), n, _p(d_x), ctx.stream()))
    return d_x


def _encodings(joiner, pts, views):
    """The fp16 encodings as the forward kernel multiplied them ([n,64] / [n,32], with their constant-1 channel right
    after the encoding; a NeRF-T net's position plane is [n,96] in the reference's column order); a view-independent net
    has no direction encoding (None)."""
    ctx = _ctx_for(pts)
    slot = ops.net_slot(joiner, ctx)
    n = pts.shape[0]
    spe = torch.empty(n, 96 if ops.is_nerft(joiner) else 64, device=pts.device, dtype=torch.float16)
    ctx.check(ctx.lib.nm_encode_f16(ctx.h, slot, 0, _p(pts), 0, n, _p(spe), ctx.stream()))
    if ops.is_viewless(joiner):
        return spe, None
    sdpe = torch.empty(n, 32, device=pts.device, dtype=torch.float16)
    ctx.check(ctx.lib.nm_encode_f16(ctx.h, slot, 1, _p(views), 0, n, _p(sdpe), ctx.stream()))
    return spe, sdpe


def _weight_grads(joiner, stash, pts, views, g, g_pre, g_f, g_v, inv):
    """dW = g^T @ layer input, K = n, fp16 operands / fp32 accumulate; g_* carry the loss scale 1/inv.
    The nine 256-wide GEMMs and their bias gradients are one k_dw_gemm launch (csrc/dw_gemm.cu).  The narrow ones
    (encodings, dL/d raw) go through cuBLAS with K split into fixed blocks (_wgrad) and whole 16-byte aligned planes
    as operands (the 64-/32-channel encodings including their padding, the [n,8]-padded dL/d raw: 63-/27-wide slices
    made cuBLAS fall back to an sm_75 kernel); the position stash's constant-1.0 channel returns pts_linears.0's bias gradient as GEMM column 63."""
    sx, sf, sv, _ = stash
    spe, sdpe = _encodings(joiner, pts, views)
    ctx = _ctx_for(g)
    n_pe = joiner.pos_pe.out_dim                                          # 63 (NeRF-T: 84): the 1.0 channel sits right after
    grads = {}
    g8 = torch.zeros(g.shape[0], 8, device=g.device, dtype=torch.float16)
    g8[:, :4] = g * (1.0 / inv)
    if ops.is_viewless(joiner):
        # output_linear (models/vanilla.py:146) reads layer 7's output: g^T @ X7 in cuBLAS, as alpha_linear below
        grads['output_linear.weight'] = _wgrad(g8, sx[7])[:4] * inv
        grads['output_linear.bias'] = g.sum(0)
    else:
        n_dpe = joiner.dir_pe.out_dim                                     # 27
        grads['rgb_linear.weight'] = _wgrad(g8, sv)[:3] * inv
        grads['rgb_linear.bias'] = g[:, :3].sum(0)
        grads['alpha_linear.weight'] = _wgrad(g8, sx[7])[3:4] * inv
        grads['alpha_linear.bias'] = g[:, 3].sum().reshape(1)
    w0 = _wgrad(g_pre[0], spe) * inv                                   # [256,64]: column 63 (84) = bias gradient (1.0 channel)
    dw, db = _dw_kernel(ctx, g_pre, g_f, g_v, sx, sf, g.shape[0])
    dw, db = dw * inv, db * inv
    if sdpe is not None:
        wd = _wgrad(g_v, sdpe) * inv                                   # [128, 32]
        grads['views_linears.0.weight'] = torch.cat([dw[8, :128], wd[:, :n_dpe]], 1)
        grads['views_linears.0.bias'] = db[8, :128]
        grads['feature_linear.weight'], grads['feature_linear.bias'] = dw[7], db[7]
    for l in range(8):
        if l == 0:
            w = w0[:, :n_pe]
        elif l == 5:
            w = torch.cat([_wgrad(g_pre[5], spe)[:, :n_pe] * inv, dw[4]], 1)
        else:
            w = dw[l - 1]
        grads['pts_linears.%d.weight' % l] = w
        grads['pts_linears.%d.bias' % l] = w0[:, n_pe] if l == 0 else db[l - 1]
    return grads


def _chain_kernel(joiner, P, stash, g):
    sx, sf, sv, sm = stash
    ctx = _ctx_for(g)
    slot = ops.net_slot(joiner, ctx)               # same weights as the forward: same slot (or an identical repack)
    n = g.shape[0]
    scale = _pow2_scale(g, 256.0)
    h = dict(device=g.device, dtype=torch.float16)
    g_pre, g_f, g_v = torch.empty(8, n, 256, **h), None, None
    if not ops.is_viewless(joiner):                 # view-independent nets: no feature / views layer gradients
        g_f, g_v = torch.empty(n, 256, **h), torch.empty(n, 128, **h)
    ctx.check(ctx.lib.nm_mlp_backward(ctx.h, slot, _p(g), _p(scale), n, _p(sv), _p(sm), _p(g_pre), _p(g_f), _p(g_v),
                                      ctx.stream()))
    return g_pre, g_f, g_v, 1.0 / scale


def _dw_kernel(ctx, g_pre, g_f, g_v, sx, sf, n):
    """The nine 256-wide weight gradients and their bias gradients, still carrying the loss scale of the g planes: one
    k_dw_gemm launch (csrc/dw_gemm.cu), every gradient and stash plane read once.
    -> dw [9,256,256], db [9,256] fp32 (plane 8: rows 0..127 used).  With g_f = g_v = sf = None (a view-independent net)
    only planes 0..6 are computed."""
    dw = torch.empty(9, 256, 256, device=g_pre.device, dtype=torch.float32)
    db = torch.empty(9, 256, device=g_pre.device, dtype=torch.float32)
    ctx.check(ctx.lib.nm_dw_gemm(ctx.h, _p(g_pre), _p(g_f), _p(g_v), _p(sx), _p(sf), n, _p(dw), _p(db), ctx.stream()))
    return dw, db


def joiner_forward(joiner, input_pts, input_views=None):
    """Joiner.forward (models/vanilla.py:162-166) with gradients to the network parameters and, when they require
    grad, to input_pts / input_views.  A view-independent net ignores input_views (may be None); its gradient is None.
    A NeRF-T net takes input_pts [...,4] = (x, y, z, t); its inputs get no gradient (nothing in the reference
    differentiates through them)."""
    nerft = ops.is_nerft(joiner)
    if nerft and (input_pts.requires_grad or (input_views is not None and input_views.requires_grad)):
        raise NotImplementedError("input gradients of NeRF-T nets (ablate_nerft) are not built")
    shape = input_pts.shape[:-1]
    pts = input_pts.float().contiguous().reshape(-1, 4 if nerft else 3)   # autograd-tracked views of the inputs
    views = None
    if not ops.is_viewless(joiner):
        views = input_views.to(pts.device).float().contiguous().reshape(-1, 3)
        assert views.shape[0] == pts.shape[0], "input_views must match input_pts"
    params = [p for _, p in joiner.nerf.named_parameters()]
    return _JoinerMLP.apply(pts, views, joiner, *params).reshape(*shape, 4)


# ---------------------------------------------------------------------------------------------
# Human trainer: differentiable observation -> canonical map and SMPL scene transforms (csrc/human_train.cu, smpl.cu)
# ---------------------------------------------------------------------------------------------
def _faces_i32(faces, device):
    return ops.faces_device(faces, device)


class _WarpDiffTinv(torch.autograd.Function):
    """T_interp_inv of utils/ray_utils.py:72-91 with gradients to the posed vertices and the per-vertex transforms."""

    @staticmethod
    def forward(fctx, verts, T, f_id, closest, faces):
        v, t = _f32(verts), _f32(T, verts.device).reshape(-1, 16)
        ctx = _ctx_for(v)
        n = int(f_id.shape[0])
        Tinv = torch.empty(n, 4, 4, device=v.device)
        with torch.cuda.device(v.device):
            ctx.check(ctx.lib.nm_warp_diff_forward(ctx.h, _p(f_id), _p(closest), _p(v), _p(faces), _p(t), n, _p(Tinv), ctx.stream()))
        fctx.save_for_backward(v, t, f_id, closest, faces)
        fctx.t_shape = tuple(T.shape)
        return Tinv

    @staticmethod
    def backward(fctx, g):
        v, t, f_id, closest, faces = fctx.saved_tensors
        ctx = _ctx_for(v)
        need_v, need_t = fctx.needs_input_grad[0], fctx.needs_input_grad[1]
        g_T = torch.empty_like(t) if need_t else None
        g_v = torch.empty_like(v) if need_v else None
        if need_v or need_t:
            with torch.cuda.device(v.device):
                ctx.check(ctx.lib.nm_warp_diff_backward(ctx.h, _p(f_id), _p(closest), _p(v), _p(faces), _p(t), int(f_id.shape[0]),
                                                        _p(_f32(g, v.device)), int(v.shape[0]), _p(g_T), _p(g_v), ctx.stream()))
        return g_v, (g_T.reshape(fctx.t_shape) if need_t else None), None, None, None


def warp_diff_tinv(verts, T, f_id, closest, faces):
    """verts [V,3], T [V,4,4] CUDA float32 (may require grad); f_id [n] int32, closest [n,3] float64 CUDA (the
    nm_signed_distance query); faces [F,>=3].  -> T_interp_inv [n,4,4]."""
    return _WarpDiffTinv.apply(verts, T, f_id.contiguous(), closest.contiguous(), _faces_i32(faces, verts.device))


class _HumanCanonicalize(torch.autograd.Function):
    """trainers/human_nerf_trainer.py:263-276 fused: (can_pts, can_dirs) from the samples, with gradients to the posed
    vertices, the per-vertex transforms and the offset."""

    @staticmethod
    def forward(fctx, verts, T, offset, pts, f_id, closest, faces):
        v, t, p = _f32(verts), _f32(T, verts.device).reshape(-1, 16), _f32(pts, verts.device)
        off = _f32(offset, v.device) if offset is not None else None
        ctx = _ctx_for(v)
        R, S = int(p.shape[0]), int(p.shape[1])
        cp, cd = torch.empty(R, S, 3, device=v.device), torch.empty(R, S, 3, device=v.device)
        with torch.cuda.device(v.device):
            ctx.check(ctx.lib.nm_human_canonicalize(ctx.h, _p(f_id), _p(closest), _p(v), _p(faces), _p(t), _p(p), _p(off), R, S,
                                                    _p(cp), _p(cd), ctx.stream()))
        fctx.save_for_backward(v, t, p, cp, f_id, closest, faces)
        fctx.t_shape = tuple(T.shape)
        return cp, cd

    @staticmethod
    def backward(fctx, g_cp, g_cd):
        v, t, p, cp, f_id, closest, faces = fctx.saved_tensors
        ctx = _ctx_for(v)
        need_v, need_t, need_o = fctx.needs_input_grad[:3]
        R, S = int(p.shape[0]), int(p.shape[1])
        g_off = torch.empty_like(p)
        g_T = torch.empty_like(t) if need_t else None
        g_v = torch.empty_like(v) if need_v else None
        g_cp = _f32(g_cp, v.device) if g_cp is not None else None
        g_cd = _f32(g_cd, v.device) if g_cd is not None else None
        with torch.cuda.device(v.device):
            ctx.check(ctx.lib.nm_human_canonicalize_backward(ctx.h, _p(f_id), _p(closest), _p(v), _p(faces), _p(t), _p(p), _p(cp),
                                                             _p(g_cp), _p(g_cd), R, S, int(v.shape[0]), _p(g_off), _p(g_T),
                                                             _p(g_v), ctx.stream()))
        return g_v, (g_T.reshape(fctx.t_shape) if need_t else None), (g_off if need_o else None), None, None, None, None


def human_canonicalize(pts, verts, T, f_id, closest, faces, offset=None):
    """pts [R,S,3] (constants), verts [V,3], T [V,4,4], offset [R,S,3] or None (may require grad) -> (can_pts, can_dirs)."""
    assert pts.dim() == 3 and pts.shape[-1] == 3 and pts.shape[1] >= 2, "pts must be [rays, samples >= 2, 3]"
    return _HumanCanonicalize.apply(verts, T, offset, pts.detach(), f_id.contiguous(), closest.contiguous(),
                                    _faces_i32(faces, verts.device))


class _VertexForward(torch.autograd.Function):
    """HumanNeRF.vertex_forward (models/human_nerf.py:92-122) with gradients to pose, betas and alignment."""

    @staticmethod
    def forward(fctx, pose, betas, alignment, da_pose, model, scale):
        dev = model.device
        p, b, a, da = (_f32(x, dev).reshape(-1) for x in (pose, betas, alignment, da_pose))
        ctx = _ctx_for(p)
        nv = model.n_verts
        T, world = torch.empty(nv, 4, 4, device=dev), torch.empty(nv, 3, device=dev)
        with torch.cuda.device(dev):
            ctx.check(ctx.lib.nm_smpl_scene_forward_train(ctx.h, C.byref(model.struct), _p(p), _p(da), _p(b), _p(a), float(scale),
                                                          _p(T), _p(world), ctx.stream()))
        fctx.save_for_backward(p, b, a, da)
        fctx.model, fctx.scale = model, float(scale)
        fctx.shapes = (tuple(pose.shape), tuple(betas.shape), tuple(alignment.shape))
        return world[None], T[None]

    @staticmethod
    def backward(fctx, g_world, g_T):
        p, b, a, da = fctx.saved_tensors
        model = fctx.model
        ctx = _ctx_for(p)
        g_world = _f32(g_world, p.device) if g_world is not None else None
        g_T = _f32(g_T, p.device) if g_T is not None else None
        gp, gb, ga = torch.empty_like(p), torch.empty_like(b), torch.empty_like(a)
        with torch.cuda.device(p.device):
            ctx.check(ctx.lib.nm_smpl_scene_backward(ctx.h, C.byref(model.struct), _p(p), _p(da), _p(b), _p(a), fctx.scale, _p(g_T),
                                                     _p(g_world), _p(gp), _p(gb), _p(ga), ctx.stream()))
        sp, sb, sa = fctx.shapes
        return gp.reshape(sp), gb.reshape(sb), ga.reshape(sa), None, None, None


def vertex_forward(model, pose, betas, alignment, scale, da_pose):
    """model: ops.SmplModelDevice; pose [1,3J], betas [1,NB], alignment [4,4] (self.alignments[idx]), da_pose [1,3J] CUDA
    tensors -> (world_verts [1,V,3], T_da2scene [1,V,4,4]) float32 with gradients to pose / betas / alignment."""
    return _VertexForward.apply(pose, betas, alignment, da_pose, model, scale)
