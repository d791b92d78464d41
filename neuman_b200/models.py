"""Host-side mirror of the reference's network containers (models/vanilla.py:17-250,
models/human_nerf.py:20-90): same class names, constructor arguments, parameter names and shapes, so
reference checkpoints (`coarse_model_state_dict`, `hybrid_model_state_dict`, ...) load unchanged.
`forward()` runs the CUDA path; under autograd it runs the training kernel (activation stash) and returns
gradients to the network parameters (neuman_b200/autograd.py, SURVEY.md §8f-1).
"""
import copy

import numpy as np
import torch
import torch.nn as nn

from . import ops


class Embedder(nn.Module):
    """models/vanilla.py:17-92. Holds only the description; the encoding itself is fused into the
    MLP kernels (csrc/nm_pe.cuh)."""

    def __init__(self, input_dims, max_freq, N_freqs, log_sampling=True, include_input=True, min_freq=0,
                 mapping='posenc'):
        super().__init__()
        if mapping not in ('posenc', 'rotate'):
            raise ValueError(mapping)
        if not log_sampling or not include_input:
            raise NotImplementedError("only log_sampling=True, include_input=True (the reference defaults)")
        self.input_dims = input_dims
        self.max_freq = max_freq
        self.min_freq = min_freq
        self.N_freqs = N_freqs
        self.log_sampling = log_sampling
        self.include_input = include_input
        self.mapping = mapping
        self.out_dim = input_dims + 2 * input_dims * N_freqs if mapping == 'posenc' else 3 + 6 * N_freqs

    def rotate_bvals(self, device=None):
        """The 'rotate' frequency matrix [3 N, 3] (models/vanilla.py:44-58): axis-aligned frequencies rotated by 45 degrees
        about z, then by 45 degrees about x; built in float64 and rounded to float32 like the reference."""
        b = 2.0 ** np.linspace(self.min_freq, self.max_freq, num=self.N_freqs)
        b = np.reshape(np.eye(3) * b[:, None, None], [len(b) * 3, 3])
        h = (2 ** .5) / 2
        b = b @ np.array([[h, -h, 0], [h, h, 0], [0, 0, 1]]).T
        b = b @ np.array([[1, 0, 0], [0, h, -h], [0, h, h]]).T
        return torch.from_numpy(b).float().to(device)

    def forward(self, inputs, cur_iter=None):
        """models/vanilla.py:82-92 as stand-alone torch ops (any device).  The renderers and trainers never call it: inside
        `Joiner.forward` / `OffsetNet.forward` the encoding is produced by the MLP kernels' own encoding warps (csrc/nm_pe.cuh).
        It exists so that code written against the reference's module interface keeps working."""
        if self.mapping == 'rotate':
            assert inputs.shape[-1] == 3
            proj = inputs @ self.rotate_bvals(inputs.device).T
            return torch.cat([inputs, torch.sin(proj), torch.cos(proj)], -1)
        assert cur_iter is None
        out = [inputs]
        for f in 2.0 ** torch.linspace(self.min_freq, self.max_freq, steps=self.N_freqs):
            out += [torch.sin(inputs * f), torch.cos(inputs * f)]
        return torch.cat(out, -1)


class NeRF(nn.Module):
    """Parameter container with the reference's module names and shapes (models/vanilla.py:95-118):
    pts_linears.{0..depth-1}, views_linears.0, feature_linear, alpha_linear, rgb_linear (or output_linear).
    Modules are created in the reference's order so a seeded default init reproduces its weights."""

    def __init__(self, depth=8, width=256, input_ch=3, input_ch_views=3, output_ch=4, skips=[4], use_viewdirs=False,
                 scale=1.0, scale_type='no'):
        super().__init__()
        self.depth, self.width = depth, width
        self.input_ch, self.input_ch_views = input_ch, input_ch_views
        self.skips, self.use_viewdirs = skips, use_viewdirs
        self.scale, self.scale_type = scale, scale_type
        trunk = []
        fan_in = input_ch
        for layer in range(depth):
            trunk.append(nn.Linear(fan_in, width))
            # the layer after a skip index sees [encoded input, hidden] (input first, models/vanilla.py:131)
            fan_in = width + input_ch if layer in self.skips else width
        self.pts_linears = nn.ModuleList(trunk)
        if not use_viewdirs:
            self.output_linear = nn.Linear(width, output_ch)
            return
        self.views_linears = nn.ModuleList([nn.Linear(width + input_ch_views, width // 2)])
        self.feature_linear = nn.Linear(width, width)
        self.alpha_linear = nn.Linear(width, 1)
        self.rgb_linear = nn.Linear(width // 2, 3)

    def forward(self, input_pts, input_views=None):
        """models/vanilla.py:120-152 on ALREADY ENCODED inputs, as library GEMMs (torch.nn.functional.linear; any device).
        The product path never takes it -- `Joiner.forward` runs encoding + network as one tensor-core kernel -- it serves code
        that drives the reference's module interface layer by layer."""
        import torch.nn.functional as F
        assert input_pts.shape[-1] == self.input_ch
        h = input_pts
        for i, lin in enumerate(self.pts_linears):
            h = F.relu(lin(h))
            if i in self.skips:
                h = torch.cat([input_pts, h], -1)
        if self.use_viewdirs:
            assert input_views is not None and input_views.shape[-1] == self.input_ch_views
            alpha = self.alpha_linear(h)
            h = torch.cat([self.feature_linear(h), input_views], -1)
            for lin in self.views_linears:
                h = F.relu(lin(h))
            out = torch.cat([self.rgb_linear(h), alpha], -1)
        else:
            out = self.output_linear(h)
        if self.scale_type == 'no':
            return out
        if self.scale_type == 'linear':
            return out * self.scale
        if self.scale_type == 'tanh':
            return torch.tanh(out) * self.scale
        raise ValueError(self.scale_type)


class Joiner(nn.Module):
    """models/vanilla.py:155-166."""

    def __init__(self, pos_pe, dir_pe, nerf):
        super().__init__()
        self.pos_pe, self.dir_pe, self.nerf = pos_pe, dir_pe, nerf

    def forward(self, input_pts, input_views=None):
        """input_pts [...,3], input_views [...,3] -> [...,4] = (r,g,b,sigma). CUDA only.  A view-independent net
        (use_viewdirs=False) ignores input_views, which may be None.
        Under autograd (a network parameter or an input requiring grad) the training kernel runs and the result
        carries gradients to the parameters and to input_pts / input_views (neuman_b200/autograd.py)."""
        if torch.is_grad_enabled() and (input_views is not None or not self.nerf.use_viewdirs) and (
                any(p.requires_grad for p in self.nerf.parameters())
                or any(isinstance(t, torch.Tensor) and t.requires_grad for t in (input_pts, input_views))):
            from . import autograd
            return autograd.joiner_forward(self, input_pts, input_views)
        return ops.joiner_forward(self, input_pts, input_views)


def build_nerf(opt):
    """models/vanilla.py:208-250."""
    mapping = opt.posenc if hasattr(opt, 'posenc') else 'posenc'
    pos_pe = Embedder(opt.raw_pos_dim, opt.pos_max_freq, opt.pos_N_freqs, opt.log_sampling, opt.include_input,
                      min_freq=opt.pos_min_freq, mapping=mapping)
    dir_pe = Embedder(opt.raw_dir_dim, opt.dir_max_freq, opt.dir_N_freqs, opt.log_sampling, opt.include_input,
                      mapping=mapping)

    def one():
        return Joiner(pos_pe, dir_pe, NeRF(depth=opt.nerf_depth, width=opt.nerf_width, input_ch=pos_pe.out_dim,
                                           input_ch_views=dir_pe.out_dim, use_viewdirs=opt.use_viewdirs))
    coarse, fine = one(), one()
    if opt.use_cuda:
        coarse, fine = coarse.cuda(), fine.cuda()
    return coarse, fine


class OffsetNet(nn.Module):
    """models/vanilla.py:169-177: one offset network (Embedder over (x, y, z, t) + an 8x256 NeRF trunk with
    `output_linear` [3,256] and output scaling); parameter names and shapes are the reference's, so
    `hybrid_model_state_dict` checkpoints load unchanged.  It is a training-time network
    (trainers/human_nerf_trainer.py:259-261); the renderers never evaluate it (SURVEY.md §0.4).

    Tensor-core path.  Inside one training step the time input is ONE number for the whole batch (`cur_view_f`, :260), and
    the trunk is the Joiner's trunk.  For a fixed t the network is therefore exactly a Joiner on (x, y, z):
      * the 21 time channels of the 84-channel encoding are constants: their products with the layer-0 / skip-layer
        weight columns fold into those layers' biases, the 63 spatial channels are the Joiner's position encoding;
      * `output_linear` (3 x 256, any sign) is carried through the Joiner's non-negative head as y = relu(y) - relu(-y):
        feature rows 0..2 = +W_o, 3..5 = -W_o, a unit views layer, rgb = [I, -I].
    `forward_at_time` builds those weights with differentiable torch indexing (a few 256-wide tensors), runs the SAME
    wgmma training / inference kernels as every other network (k_mlp_tc, k_mlp_tc_bwd, k_dw_gemm), and autograd carries
    the Joiner-shaped gradients back to this module's parameters.  `forward` uses it when the time column is constant and
    the architecture is the reference's default (8 x 256, skip 4, 10 log-spaced frequencies); otherwise it evaluates the
    network with library GEMMs (torch.nn.functional.linear, float32), which is also the CPU path."""

    def __init__(self, pos_pe, nerf):
        super().__init__()
        self.pos_pe, self.nerf = pos_pe, nerf

    # ---- library path ------------------------------------------------------------------------------------------
    def encode(self, x):
        """Embedder.forward, mapping 'posenc' (models/vanilla.py:60-79,90-92): [x, sin(f0 x), cos(f0 x), sin(f1 x), ...]."""
        if self.pos_pe.mapping != 'posenc':
            raise NotImplementedError("offset nets use the 'posenc' mapping (models/vanilla.py:180-188)")
        out = [x]
        for f in _offset_freqs(self, x.device):
            out += [torch.sin(x * f), torch.cos(x * f)]
        return torch.cat(out, -1)

    def forward_library(self, input_pts):
        import torch.nn.functional as F
        n = self.nerf
        e = self.encode(input_pts)
        h = e
        for i, lin in enumerate(n.pts_linears):                         # NeRF.forward, use_viewdirs=False (:127-152)
            h = F.relu(lin(h))
            if i in n.skips:
                h = torch.cat([e, h], -1)
        return _offset_scaled(self, n.output_linear(h))

    # ---- tensor-core path (module-level functions below: they also serve the reference's own OffsetNet instances) ----
    def tc_supported(self):
        return offset_tc_supported(self)

    def joiner_weights(self, t):
        return offset_joiner_weights(self, t)

    def forward_at_time(self, pts, t):
        """pts [...,3] CUDA, t: the step's time (float or 0-d tensor) -> offsets [...,3] on the tensor-core kernels."""
        return offset_forward_at_time(self, pts, t)

    def forward(self, input_pts, cur_iter=None):
        assert cur_iter is None                                          # (:91)
        out = offset_forward_tc_if_constant_time(self, input_pts)
        return self.forward_library(input_pts) if out is None else out


def _offset_freqs(net, device=None):
    pe = net.pos_pe
    return 2.0 ** torch.linspace(pe.min_freq, pe.max_freq, steps=pe.N_freqs, device=device)


def _offset_scaled(net, out):
    n = net.nerf
    if n.scale_type == 'no':
        return out
    if n.scale_type == 'linear':
        return out * n.scale
    if n.scale_type == 'tanh':
        return torch.tanh(out) * n.scale
    raise ValueError(n.scale_type)


def offset_tc_supported(net):
    """True for the reference's default offset-net architecture (models/vanilla.py:180-205 with options/options.py defaults)."""
    try:
        n, pe = net.nerf, net.pos_pe
        return bool(pe.mapping == 'posenc' and pe.input_dims == 4 and pe.N_freqs == 10 and pe.log_sampling and pe.include_input
                    and len(n.pts_linears) == 8 and tuple(n.pts_linears[1].weight.shape) == (256, 256)
                    and tuple(n.skips) == (4,) and not n.use_viewdirs and tuple(n.output_linear.weight.shape) == (3, 256))
    except AttributeError:
        return False


def offset_channel_split(n_freqs):
    """Indices of the 63 spatial and the 21 time channels inside the 84-channel encoding of (x, y, z, t)
    (models/vanilla.py:60-79: identity, then sin and cos of all four inputs per frequency)."""
    xyz, tt = [0, 1, 2], [3]
    for k in range(n_freqs):
        s, c = 4 + 8 * k, 4 + 8 * k + 4
        xyz += [s, s + 1, s + 2, c, c + 1, c + 2]
        tt += [s + 3, c + 3]
    return xyz, tt


def _offset_consts(net, dev):
    """Per-device constants of the Joiner form (index lists, frequencies, the fixed head weights): built once and kept
    on the instance, so that a training step issues no host->device copy for them."""
    pe = net.pos_pe
    key = (str(dev), int(pe.N_freqs), float(pe.min_freq), float(pe.max_freq))
    cache = net.__dict__.setdefault('_nm_consts', {})
    c = cache.get(key)
    if c is None:
        with torch.inference_mode(False), torch.no_grad():
            xyz, tt = offset_channel_split(pe.N_freqs)
            vw = torch.zeros(128, 256 + 27)
            vw[torch.arange(6), torch.arange(6)] = 1.0
            rw = torch.zeros(3, 128)
            rw[torch.arange(3), torch.arange(3)] = 1.0
            rw[torch.arange(3), torch.arange(3) + 3] = -1.0
            c = {'xyz': torch.tensor(xyz).to(dev), 'tt': torch.tensor(tt).to(dev),
                 'freqs': (2.0 ** torch.linspace(pe.min_freq, pe.max_freq, steps=pe.N_freqs)).to(dev),
                 'pad_w': torch.zeros(250, 256).to(dev), 'pad_b': torch.zeros(250).to(dev),
                 'alpha_w': torch.zeros(1, 256).to(dev), 'alpha_b': torch.zeros(1).to(dev),
                 'views_w': vw.to(dev), 'views_b': torch.zeros(128).to(dev), 'rgb_w': rw.to(dev), 'rgb_b': torch.zeros(3).to(dev)}
        cache.clear()                                          # one device at a time is all a module lives on
        cache[key] = c
    return c


def offset_joiner_weights(net, t):
    """The Joiner-shaped parameters equivalent to offset network `net` at time t (0-d tensor or float), as differentiable
    functions of its parameters; keys = NeRF(use_viewdirs=True).named_parameters() names."""
    n = net.nerf
    dev = n.output_linear.weight.device
    c = _offset_consts(net, dev)
    xyz_i, tt_i = c['xyz'], c['tt']
    if isinstance(t, torch.Tensor):
        t = t.detach().to(device=dev, dtype=torch.float32).reshape(())
    else:
        t = torch.full((), float(t), dtype=torch.float32, device=dev)          # a fill kernel: no host->device copy
    ft = t * c['freqs']
    pe_t = torch.cat([t[None], torch.stack([torch.sin(ft), torch.cos(ft)], 1).reshape(-1)])      # [t, sin f0 t, cos f0 t, sin f1 t, ...]
    n_in = net.pos_pe.out_dim                                        # 84
    W = {}
    for l, lin in enumerate(n.pts_linears):
        w, b = lin.weight, lin.bias
        if l == 0:
            W['pts_linears.0.weight'] = w[:, xyz_i]
            W['pts_linears.0.bias'] = b + w[:, tt_i] @ pe_t
        elif (l - 1) in n.skips:
            W[f'pts_linears.{l}.weight'] = torch.cat([w[:, xyz_i], w[:, n_in:]], 1)
            W[f'pts_linears.{l}.bias'] = b + w[:, tt_i] @ pe_t
        else:
            W[f'pts_linears.{l}.weight'], W[f'pts_linears.{l}.bias'] = w, b
    wo, bo = n.output_linear.weight, n.output_linear.bias
    W['feature_linear.weight'] = torch.cat([wo, -wo, c['pad_w']], 0)
    W['feature_linear.bias'] = torch.cat([bo, -bo, c['pad_b']])
    W['alpha_linear.weight'], W['alpha_linear.bias'] = c['alpha_w'], c['alpha_b']
    W['views_linears.0.weight'], W['views_linears.0.bias'] = c['views_w'], c['views_b']
    W['rgb_linear.weight'], W['rgb_linear.bias'] = c['rgb_w'], c['rgb_b']
    return W


def offset_shadow_joiner(net):
    """The Joiner module whose parameters receive offset_joiner_weights() before every launch (the kernels pack from
    it).  Kept in the instance dict inside a tuple so that it never shows up among the offset net's own parameters."""
    dev = net.nerf.output_linear.weight.device
    sh = net.__dict__.get('_nm_shadow')
    if sh is None or next(sh[0].parameters()).device != dev:
        pe = net.pos_pe
        pos = Embedder(3, pe.max_freq, pe.N_freqs, pe.log_sampling, pe.include_input, min_freq=pe.min_freq)
        dpe = Embedder(3, 3, 4, True, True)
        j = Joiner(pos, dpe, NeRF(depth=8, width=256, input_ch=pos.out_dim, input_ch_views=dpe.out_dim, use_viewdirs=True)).to(dev)
        for p in j.parameters():
            p.requires_grad_(False)
        sh = (j,)
        net.__dict__['_nm_shadow'] = sh
    return sh[0]


def offset_forward_at_time(net, pts, t):
    from . import autograd
    j = offset_shadow_joiner(net)
    W = offset_joiner_weights(net, t)
    names = [k for k, _ in j.nerf.named_parameters()]
    with torch.no_grad():
        for k, p in j.nerf.named_parameters():
            p.copy_(W[k])
    shape = pts.shape[:-1]
    x = pts.detach().float().reshape(-1, 3).contiguous()
    views = torch.zeros_like(x)
    if torch.is_grad_enabled() and any(p.requires_grad for p in net.nerf.parameters()):
        raw = autograd._JoinerMLP.apply(x, views, j, *[W[k] for k in names])
    else:
        raw = ops.joiner_forward(j, x, views)
    return _offset_scaled(net, raw[:, :3]).reshape(*shape, 3)


def offset_forward_tc_if_constant_time(net, input_pts):
    """OffsetNet.forward on the tensor-core path when it applies: CUDA input [...,4] whose time column is one value (what
    trainers/human_nerf_trainer.py:260 builds) and the default architecture.  Returns None otherwise.  The constancy check
    is one host read per call; callers that know the step's time use forward_at_time / offset_forward_at_time directly."""
    if not (isinstance(input_pts, torch.Tensor) and input_pts.is_cuda and input_pts.shape[-1] == 4 and input_pts.numel()
            and offset_tc_supported(net) and net.nerf.output_linear.weight.is_cuda):
        return None
    tcol = input_pts[..., 3]
    t0 = tcol.reshape(-1)[0]
    if not bool((tcol == t0).all()):
        return None
    return offset_forward_at_time(net, input_pts[..., :3], t0.detach())


def build_offset_net(opt):
    """models/vanilla.py:180-205."""
    st_pe = Embedder(opt.raw_pos_dim + 1, opt.pos_max_freq, opt.pos_N_freqs, opt.log_sampling, opt.include_input,
                     min_freq=opt.pos_min_freq)
    net = NeRF(depth=opt.nerf_depth, width=opt.nerf_width, input_ch=st_pe.out_dim, input_ch_views=0, output_ch=3,
               use_viewdirs=False, scale=opt.offset_scale, scale_type=opt.offset_scale_type)
    net = OffsetNet(st_pe, net)
    return net.cuda() if opt.use_cuda else net


class SMPL(nn.Module):
    """Device mirror of the part of models/smpl.py:SMPL the path uses: `verts_transformations` (:109-162) and `forward`
    (:164-215) on the CUDA LBS kernels (csrc/smpl.cu).  `model`: a path to an SMPL pickle (the reference's
    data/smplx/smpl/SMPL_NEUTRAL.pkl layout: f, v_template, shapedirs, J_regressor, posedirs, kintree_table, weights)
    or a dict with those keys (neuman_b200.synthetic.make_model())."""

    def __init__(self, model, device="cuda"):
        super().__init__()
        if isinstance(model, str):
            import pickle
            with open(model, "rb") as fp:
                model = pickle.load(fp, encoding="latin1")
        dense = lambda a: np.asarray(a.todense() if hasattr(a, "todense") else a)
        self.faces = np.asarray(model["f"]).astype(np.int64)
        par = np.asarray(model["kintree_table"])[0].astype(np.int64)
        self.device = torch.device(device)
        self.dev_model = ops.SmplModelDevice(dense(model["v_template"]), dense(model["shapedirs"])[:, :, :10],
                                             dense(model["J_regressor"]), dense(model["weights"]), par, device=self.device)

    def verts_transformations(self, poses, betas, transl=None, return_tensor=True, concat_joints=False):
        """-> (vertices [1,V(+J),3], T [1,V(+J),4,4]) float32 (numpy [V,3] / [V,4,4] when return_tensor=False)."""
        verts, T = ops.smpl_verts_transformations(self.dev_model, poses, betas, concat_joints=concat_joints)
        if transl is not None:
            T = T.clone()
            T[:, :3, 3] += torch.as_tensor(transl, dtype=torch.float32, device=T.device).reshape(1, 3)   # transl_4x4 @ L (:151-154)
        if not return_tensor:
            return verts.cpu().numpy(), T.cpu().numpy()
        return verts[None], T[None]

    def forward(self, poses, betas, transl=None, return_tensor=True, return_joints=False):
        """SMPL.forward (:164-215): posed vertices = T . [v_shaped; 1] (pose blend shapes are not applied, :334)."""
        verts, T = ops.smpl_verts_transformations(self.dev_model, poses, betas, concat_joints=True)
        posed = torch.einsum("vij,vj->vi", T[:, :3, :3], verts) + T[:, :3, 3]
        if transl is not None:
            posed = posed + torch.as_tensor(transl, dtype=torch.float32, device=posed.device).reshape(1, 3)
        nv = self.dev_model.n_verts
        v, j = posed[:nv], posed[nv:]
        if not return_tensor:
            v, j = v.cpu().numpy(), j.cpu().numpy()
        else:
            v, j = v[None], j[None]
        return (v, j) if return_joints else v


class HumanNeRF(nn.Module):
    """models/human_nerf.py:20-122: container of the background coarse/fine nets, the offset nets and the canonical human
    net, plus -- when per-frame SMPL parameters are given -- `poses / betas / alignments / scale`, the `body_model`, the
    'da' rest pose and `vertex_forward`.  `smpl_model`: path or dict for the body model (the reference hard-codes
    <repo>/data/smplx/smpl/SMPL_NEUTRAL.pkl, which is licence-gated and absent here)."""

    def __init__(self, opt, poses=None, betas=None, alignments=None, scale=None, smpl_model=None):
        super().__init__()
        self.coarse_bkg_net, self.fine_bkg_net = build_nerf(opt)
        self.offset_nets = nn.ModuleList([build_offset_net(opt) for _ in range(getattr(opt, "num_offset_nets", 0))])
        t = copy.deepcopy(opt)
        t.pos_min_freq = 0
        t.use_viewdirs = t.specular_can
        t.posenc = t.can_posenc
        self.coarse_human_net, _ = build_nerf(t)
        self.body_model = None
        if poses is not None:
            assert betas is not None and alignments is not None and scale is not None
            dev = "cuda" if opt.use_cuda else "cpu"
            self.poses = nn.Parameter(torch.from_numpy(np.asarray(poses)).float().to(dev))
            self.betas = nn.Parameter(torch.from_numpy(np.asarray(betas)).float().to(dev))
            self.alignments = nn.Parameter(torch.from_numpy(np.asarray(alignments)).float().to(dev))
            self.scale = scale
            da = torch.zeros(self.poses.shape[1] // 3, 3)
            da[1, 2], da[2, 2] = 1.0, -1.0                                   # (:46-50)
            self.da_smpl = nn.Parameter(da.reshape(1, -1).to(dev), requires_grad=False)
            self.poses_orig, self.betas_orig = np.array(poses, copy=True), np.array(betas, copy=True)
            if smpl_model is not None:
                self.body_model = SMPL(smpl_model, device="cuda")

    def vertex_forward(self, idx, pose=None, beta=None):
        """models/human_nerf.py:92-122 -> (world_verts [1,V,3] f32, T_da2scene [1,V,4,4] f32) on the device.
        Without autograd: one nm_smpl_scene_transforms call (LBS of the frame pose and of the 'da' pose,
        T_t2pose . inv(T_t2da), alignment^T and the scene scale; float64 inside like data_io/neuman_helper.py:299-330,
        returned in the reference's float32).  Under autograd (the human trainer optimises poses / betas / alignments,
        trainers/human_nerf_trainer.py:263): the float32 training kernels, whose adjoint returns the gradients of those
        three parameters (neuman_b200.autograd.vertex_forward)."""
        if self.body_model is None:
            raise RuntimeError("HumanNeRF was built without an SMPL model (pass smpl_model=...)")
        pose = self.poses[idx][None] if pose is None else pose
        beta = self.betas[idx][None] if beta is None else beta
        m = self.body_model.dev_model
        if torch.is_grad_enabled() and any(t.requires_grad for t in (pose, beta, self.alignments)):
            from . import autograd
            return autograd.vertex_forward(m, pose, beta, self.alignments[idx], float(self.scale), self.da_smpl)
        world, _, T = ops.smpl_scene_transforms(m, pose.detach(), beta.detach(), self.alignments[idx].detach().cpu().numpy(),
                                                float(self.scale))
        return world[None], T[:m.n_verts].float()[None]


def default_opt(**over):
    """options/options.py:52-81 defaults consumed by the path."""
    import types
    o = types.SimpleNamespace(
        use_cuda=torch.cuda.is_available(), nerf_depth=8, nerf_width=256, use_viewdirs=True, specular_can=True,
        raw_pos_dim=3, pos_min_freq=0, pos_max_freq=9, pos_N_freqs=10, raw_dir_dim=3, dir_max_freq=3, dir_N_freqs=4,
        log_sampling=True, include_input=True, can_posenc='rotate', rays_per_batch=2048, samples_per_ray=128,
        white_bkg=True, importance_samples_per_ray=128, num_offset_nets=0, offset_scale=1.0, offset_scale_type='linear')
    o.__dict__.update(over)
    return o
