"""GPU parity of the backward kernels (training path, SURVEY.md §8f-1) against torch autograd of the oracle
restatement (float32 / float64 on the CPU)."""
import numpy as np
import pytest
import torch

from neuman_b200 import autograd as nag
from oracle import neuman_oracle as no
from tests import util

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("R,S,white", [(5, 7, True), (64, 128, True), (33, 256, False), (3, 33, True)])
def test_raw2outputs_backward(R, S, white):
    torch.manual_seed(R * S)
    raw = (torch.randn(R, S, 4) * 1.5).double().requires_grad_(True)
    z = torch.sort(torch.rand(R, S) * 3, -1)[0].double()
    d = torch.randn(R, 3).double()
    noise = (torch.randn(R, S) * 0.3).double()
    # oracle in float64 for a clean reference gradient
    with torch.enable_grad():
        dz = torch.cat([z[..., 1:] - z[..., :-1], torch.full_like(z[..., :1], 1e10)], -1) * torch.linalg.norm(d[..., None, :], dim=-1)
        rgb = torch.sigmoid(raw[..., :3])
        alpha = 1. - torch.exp(-torch.relu(raw[..., 3] + noise) * dz)
        T = torch.cumprod(torch.cat([torch.ones(R, 1, dtype=torch.float64), 1. - alpha + 1e-10], -1), -1)[:, :-1]
        w = alpha * T
        rgb_map = (w[..., None] * rgb).sum(-2)
        depth, acc = (w * z).sum(-1), w.sum(-1)
        if white:
            rgb_map = rgb_map + (1. - acc[..., None])
        g_rgb, g_depth, g_acc, g_w = torch.randn(R, 3).double(), torch.randn(R).double(), torch.randn(R).double(), torch.randn(R, S).double()
        loss = (rgb_map * g_rgb).sum() + (depth * g_depth).sum() + (acc * g_acc).sum() + (w * g_w).sum()
        loss.backward()
    ref = raw.grad.float()
    raw_c = raw.detach().float().to(DEV).requires_grad_(True)
    outs = nag.raw2outputs(raw_c, z.float().to(DEV), d.float().to(DEV), raw_noise_std=1.0, white_bkg=white, noise=noise.float().to(DEV))
    l2 = (outs[0] * g_rgb.float().to(DEV)).sum() + (outs[4] * g_depth.float().to(DEV)).sum() + \
        (outs[2] * g_acc.float().to(DEV)).sum() + (outs[3] * g_w.float().to(DEV)).sum()
    l2.backward()
    got = raw_c.grad.cpu()
    scale = ref.abs().max()
    assert (got - ref).abs().max() < 2e-5 * max(1.0, float(scale)), ((got - ref).abs().max(), scale)
    # only rgb gradient (the vanilla trainer's case): other grads None
    raw_c.grad = None
    outs = nag.raw2outputs(raw_c, z.float().to(DEV), d.float().to(DEV), white_bkg=white)
    outs[0].sum().backward()
    assert torch.isfinite(raw_c.grad).all()


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


@pytest.mark.parametrize("n", [1, 63, 64, 1000, 4173, 64 * 74 * 3 + 5])
def test_dw_gemm(n):
    """k_dw_gemm (TMA-fed MN-major wgmma GEMMs, K = n) against fp32 matmuls of the same fp16 planes: fp32
    accumulation in a different order -> 1e-4 relative L2; rows 128.. of the views item stay zero."""
    from neuman_b200 import ops
    from neuman_b200.ops import _p
    torch.manual_seed(n)
    g_pre = (torch.randn(8, n, 256, device=DEV) * 0.5).half()
    g_f = (torch.randn(n, 256, device=DEV) * 0.5).half()
    g_v = (torch.randn(n, 128, device=DEV) * 0.5).half()
    sx = torch.relu(torch.randn(8, n, 256, device=DEV)).half()
    sf = torch.randn(n, 256, device=DEV).half()
    ctx = ops._ctx_for(g_f)
    out = torch.full((9, 256, 256), float("nan"), device=DEV)
    bias = torch.full((9, 256), float("nan"), device=DEV)
    ctx.check(ctx.lib.nm_dw_gemm(ctx.h, _p(g_pre), _p(g_f), _p(g_v), _p(sx), _p(sf), n, _p(out), _p(bias), ctx.stream()))
    ref = torch.zeros(9, 256, 256, device=DEV)
    for k in range(7):
        ref[k] = g_pre[k + 1].float().t() @ sx[k].float()
    ref[7] = g_f.float().t() @ sx[7].float()
    ref[8, :128] = g_v.float().t() @ sf.float()
    assert torch.isfinite(out).all()
    assert torch.equal(out[8, 128:], torch.zeros_like(out[8, 128:]))
    bref = torch.zeros(9, 256, device=DEV)
    bref[:7] = g_pre[1:].float().sum(1)
    bref[7] = g_f.float().sum(0)
    bref[8, :128] = g_v.float().sum(0)
    scale = float(bref.abs().max()) + 1.0
    assert (bias - bref).abs().max() < 1e-4 * scale, (bias - bref).abs().max()
    for k in range(9):
        assert _rel(out[k].cpu(), ref[k].cpu()) < 2e-4, (k, _rel(out[k].cpu(), ref[k].cpu()))


class _Q16(torch.autograd.Function):
    """round to fp16 in the forward, identity in the backward"""
    @staticmethod
    def forward(ctx, x):
        return x.half().float()

    @staticmethod
    def backward(ctx, gy):
        return gy


def _reference_grads(joiner, pts, views, g, quant):
    """fp32 CPU autograd of the oracle MLP.  quant=True rounds the GEMM operands (weights, encodings, layer
    outputs) to fp16 like the tensor-core path, so its ReLU masks are those of the CUDA forward."""
    import torch.nn.functional as F
    from tests.util import oracle_params
    net = oracle_params(joiner)
    for k in net.sd:
        net.sd[k].requires_grad_(True)
    if not quant:
        raw = no.net_forward(net, pts, views)
    else:
        q = _Q16.apply
        pe, ve = q(no.embed(pts, net.pos_pe)), q(no.embed(views, net.dir_pe))
        h = pe
        for i in range(8):
            pre = F.relu(F.linear(h, q(net.w(f"pts_linears.{i}.weight")), net.w(f"pts_linears.{i}.bias")))
            if i == 7:
                alpha = F.linear(pre, net.w("alpha_linear.weight"), net.w("alpha_linear.bias"))   # fp32 head
            h = q(pre)
            if i == 4:
                h = torch.cat([pe, h], -1)
        feat = q(F.linear(h, q(net.w("feature_linear.weight")), net.w("feature_linear.bias")))
        hv = q(F.relu(F.linear(torch.cat([feat, ve], -1), q(net.w("views_linears.0.weight")), net.w("views_linears.0.bias"))))
        raw = torch.cat([F.linear(hv, q(net.w("rgb_linear.weight")), net.w("rgb_linear.bias")), alpha], -1)
    (raw * g).sum().backward()
    return raw.detach(), {k[len('nerf.'):]: v.grad for k, v in net.sd.items()}


@pytest.mark.parametrize("kind", ["posenc", "rotate"])
def test_joiner_input_gradients(kind):
    """dL/d(input_pts), dL/d(input_views) (what the human trainer's differentiable warp consumes,
    trainers/human_nerf_trainer.py:266-276) against CPU autograd: fp16-operand emulation 3e-2, plain fp32 8e-2
    (same mask-flip argument as for the parameters)."""
    from tests.util import product_nets
    coarse, fine, human = product_nets(DEV)
    j = coarse if kind == "posenc" else human
    n = 3000
    torch.manual_seed(7)
    pts0 = torch.randn(n, 3) * 0.7
    views0 = torch.nn.functional.normalize(torch.randn(n, 3), dim=-1)
    g = torch.randn(n, 4)
    refs = []
    for quant in (True, False):
        p, v = pts0.clone().requires_grad_(True), views0.clone().requires_grad_(True)
        _reference_grads(j, p, v, g, quant)
        refs.append((p.grad, v.grad))
    for frozen in (False, True):                    # inputs get gradients also when the net is frozen
        for q in j.parameters():
            q.requires_grad_(not frozen)
        p, v = pts0.to(DEV).requires_grad_(True), views0.to(DEV).requires_grad_(True)
        raw = j(p, v)
        (raw * g.to(DEV)).sum().backward()
        for got, rq, rf, name in ((p.grad.cpu(), refs[0][0], refs[1][0], "pts"), (v.grad.cpu(), refs[0][1], refs[1][1], "views")):
            assert torch.isfinite(got).all()
            assert _rel(got, rq) < 3e-2, (name, "vs emulation", _rel(got, rq))
            assert _rel(got, rf) < 8e-2, (name, "vs fp32", _rel(got, rf))
    for q in j.parameters():
        q.requires_grad_(True)


@pytest.mark.parametrize("kind,n", [("posenc", 1000), ("rotate", 4096 + 77), ("posenc", 256 * 148 * 2 + 300)])
def test_joiner_backward(kind, n, monkeypatch):
    """Parameter gradients of Joiner.forward.
    (1) tensor-core backward kernel vs the same chain in torch GEMMs on the same stash: 2e-3 relative L2
        (fp16 rounding of intermediate gradients at the same points, different accumulation order);
    (2) vs fp32 CPU autograd of an fp16-operand emulation of the forward (same ReLU masks up to rare
        accumulation-order flips): 3e-2;
    (3) vs fp32 CPU autograd of the plain fp32 oracle: 8e-2 -- the fp16 operand rounding flips the sign of
        ~5e-4 of the pre-activations, and each flip changes that unit's gradient entirely (DESIGN.md
        "Training numerics"; an fp32-vs-emulation comparison on the CPU alone shows the same 2-3.5 %)."""
    from tests.util import product_nets
    coarse, fine, human = product_nets(DEV)
    j = coarse if kind == "posenc" else human
    torch.manual_seed(n)
    pts = torch.randn(n, 3) * 1.5
    views = torch.nn.functional.normalize(torch.randn(n, 3), dim=-1)
    g = torch.randn(n, 4)

    def product(torch_chain):
        if torch_chain:
            monkeypatch.setattr(nag, "_chain_kernel", util.chain_torch)
            monkeypatch.setattr(nag, "_dw_kernel", util.dw_torch)
        j.zero_grad()
        raw = j(pts.to(DEV), views.to(DEV))
        assert raw.requires_grad
        (raw * g.to(DEV)).sum().backward()
        return raw.detach().cpu(), {k: p.grad.detach().cpu().clone() for k, p in j.nerf.named_parameters()}
    raw, got = product(False)
    _, chain = product(True)
    for k in got:
        assert torch.isfinite(got[k]).all(), k
        assert _rel(got[k], chain[k]) < 2e-3, ("kernel vs torch chain", k, _rel(got[k], chain[k]))
    if n <= 5000:
        raw_q, ref_q = _reference_grads(j, pts, views, g, True)
        raw_f, ref_f = _reference_grads(j, pts, views, g, False)
        assert (raw - raw_f).abs().max() < 5e-3
        for k in got:
            assert got[k].shape == ref_f[k].shape, k
            assert _rel(got[k], ref_q[k]) < 3e-2, ("vs fp16-operand emulation", k, _rel(got[k], ref_q[k]))
            assert _rel(got[k], ref_f[k]) < 8e-2, ("vs fp32", k, _rel(got[k], ref_f[k]))
    # inference path unchanged by the training kernel: same raw under no_grad
    with torch.no_grad():
        raw2 = j(pts.to(DEV), views.to(DEV))
    assert not raw2.requires_grad and torch.equal(raw2.cpu(), raw)


def test_vanilla_train_step_matches_autograd():
    """One loss_func evaluation (trainers/vanilla_nerf_trainer.py:45-96) on the CUDA path vs the oracle's
    torch restatement under CPU autograd, sharing the stratified jitter, the density noise and the fine
    sample depths.  Then three optimizer steps on each side: losses stay together."""
    import copy
    import neuman_b200 as nb
    from neuman_b200 import train as nt
    from tests.util import product_nets, oracle_params
    import torch.nn.functional as F
    coarse, fine, _ = product_nets(DEV)
    coarse, fine = copy.deepcopy(coarse), copy.deepcopy(fine)
    opt = nb.default_opt(samples_per_ray=32, importance_samples_per_ray=32, perturb=1.0, raw_noise_std=1.0, margin=0.9)
    R = 300
    torch.manual_seed(5)
    o = torch.randn(R, 3) * 0.1
    d = torch.nn.functional.normalize(torch.randn(R, 3), dim=-1) * (1 + 0.2 * torch.rand(R, 1))
    batch = dict(origin=o.to(DEV), direction=d.to(DEV), near=torch.full((R,), 0.5, device=DEV),
                 far=torch.full((R,), 4.0, device=DEV), color=torch.rand(R, 3, device=DEV),
                 depth=(1.5 + torch.rand(R)).to(DEV))
    t_rand = torch.rand(R, 32)
    noise = (torch.randn(R, 32), torch.randn(R, 64))
    kw = dict(check_bad_weights=False, penalize_empty_space=0.1, t_rand=t_rand.to(DEV), noise=tuple(x.to(DEV) for x in noise))
    losses = nt.vanilla_loss_func(coarse, fine, batch, opt, **kw)
    sum(losses).backward()
    # reference on the CPU with the product's sample depths
    with torch.no_grad():
        _, _, z = nb.ray_to_samples(batch, 32, perturb=1.0, t_rand=t_rand.to(DEV))
        raw_c = coarse(*nb.ray_to_samples(batch, 32, perturb=1.0, t_rand=t_rand.to(DEV))[:2])
        w = nb.raw2outputs(raw_c, z, batch['direction'], raw_noise_std=1.0, white_bkg=True, noise=noise[0].to(DEV))[3]
        _, _, Fz = nb.ray_to_importance_samples(batch, z, w, 32)
    z, Fz = z.cpu(), Fz.cpu()
    nets = [oracle_params(coarse), oracle_params(fine)]
    for net in nets:
        for k in net.sd:
            net.sd[k].requires_grad_(True)

    def side(net, zz, nz):
        pts = o[:, None, :] + d[:, None, :] * zz[..., None]
        raw = no.net_forward(net, pts, d[:, None, :].expand_as(pts))
        rgb = no.raw2outputs(raw, zz, d, raw_noise_std=1.0, white_bkg=True, noise=nz)[0]
        m = zz < (batch['depth'].cpu()[:, None] * 0.9)
        s = raw[m][:, 3]
        return F.mse_loss(rgb, batch['color'].cpu()), F.l1_loss(torch.tanh(torch.relu(s)), torch.zeros_like(s)) * 0.1
    ref = side(nets[0], z, noise[0]) + side(nets[1], Fz, noise[1])
    sum(ref).backward()
    for a, b in zip(losses, (ref[0], ref[1], ref[2], ref[3])):
        assert abs(float(a) - float(b)) < 2e-4 * max(1.0, abs(float(b))), (float(a), float(b))
    for jn, net in zip((coarse, fine), nets):
        for name, p in jn.nerf.named_parameters():
            refg = net.sd['nerf.' + name].grad
            assert _rel(p.grad.cpu(), refg) < 8e-2, (name, _rel(p.grad.cpu(), refg))
    # a few optimizer steps: the loss goes down and the parameters stay finite
    optim = torch.optim.Adam(list(coarse.parameters()) + list(fine.parameters()), lr=5e-4)
    first = last = None
    for it in range(6):
        last = float(nt.train_batch(coarse, fine, optim, batch, opt, iteration=it, **kw))
        first = last if first is None else first
    assert np.isfinite(last) and last < first, (first, last)


def test_background_ray_batcher():
    """neuman_b200.data.BackgroundRayBatcher against a numpy restatement of BackgroundRayDataset.__getitem__
    (datasets/background_rays.py:56-139) on the same pixels (rays: oracle shot_rays), bit-exact except the rays
    (2e-6, as in test_gpu_stages); the random part only draws admissible pixels and fills the batch."""
    import types
    import neuman_b200 as nb
    from neuman_b200 import data as nd
    from neuman_b200.render import SimpleCapture
    rng = np.random.RandomState(3)
    caps = []
    for k in range(3):
        H, W = 48 + 8 * k, 64
        K = np.array([[60.0, 0, W / 2], [0, 60.0, H / 2], [0, 0, 1]])
        c2w = np.eye(4)
        c2w[:3, 3] = rng.normal(0, 0.2, 3)
        cap = SimpleCapture(K, c2w, H, W, near=0.3 + 0.1 * k, far=4.0 + k)
        cap.image = rng.randint(0, 256, (H, W, 3)).astype(np.uint8)
        cap.depth_map = rng.uniform(0.5, 3.0, (H, W)).astype(np.float32)
        cap.mask = (rng.uniform(size=(H, W)) < 0.3).astype(np.uint8)
        cap.binary_mask = cap.mask
        if k == 1:
            cap.border_mask = (rng.uniform(size=(H, W)) < 0.2).astype(np.uint8)
        cap.frame_id = {'frame_id': k, 'total_frames': 7}
        caps.append(cap)
    opt = types.SimpleNamespace(rays_per_batch=500, use_fused_depth=False, ablate_nerft=False)
    b = nd.BackgroundRayBatcher(opt, caps)
    np.random.seed(0)
    coords = b.sample_coords()
    assert sum(0 if c is None else c.shape[0] for c in coords) == 500
    for cap, c in zip(caps, coords):
        if c is None:
            continue
        c = c.cpu().numpy()
        bad = cap.mask[c[:, 1], c[:, 0]] != 0
        if hasattr(cap, 'border_mask'):
            bad |= cap.border_mask[c[:, 1], c[:, 0]] != 0
        assert not bad.any()
    out = b.batch_from_coords(coords)
    ref = {k: [] for k in ('color', 'depth', 'origin', 'direction', 'near', 'far', 'is_bkg', 'viewf_list')}
    for cap, c in zip(caps, coords):
        if c is None:
            continue
        c = c.cpu().numpy()
        num = c.shape[0]
        ref['color'].append((cap.image[c[:, 1], c[:, 0]] / 255).astype(np.float32))
        ref['depth'].append(cap.depth_map[c[:, 1], c[:, 0]].astype(np.float32))
        o, d = no.shot_rays(cap.intrinsic_matrix, cap.cam_pose.camera_to_world, c)
        ref['origin'].append(np.asarray(o, dtype=np.float32))
        ref['direction'].append(np.asarray(d, dtype=np.float32))
        near, far = np.stack([[cap.near['bkg']]] * num), np.stack([[cap.far['bkg']]] * num)
        ref['near'].append(near.astype(np.float32))
        ref['far'].append(far.astype(np.float32))
        ref['is_bkg'].append(np.ones_like(far).astype(np.int64))
        ref['viewf_list'].append((np.ones_like(near) * cap.frame_id['frame_id'] / cap.frame_id['total_frames']).astype(np.float32))
    for k, v in ref.items():
        r = np.concatenate(v)
        g = out[k].cpu().numpy()
        assert g.shape == r.shape and g.dtype == r.dtype, (k, g.shape, r.shape, g.dtype, r.dtype)
        if k in ('origin', 'direction'):
            assert np.abs(g - r).max() < 2e-6, k
        else:
            assert np.array_equal(g, r), k
    # the batch feeds the training step as is
    full = b()
    assert full['origin'].shape == (500, 3) and full['near'].shape == (500, 1) and full['is_bkg'].dtype == torch.long


def test_human_ray_batcher():
    """neuman_b200.data.HumanRayBatcher against a numpy restatement of HumanRayDataset.__getitem__
    (datasets/human_rays.py:145-247, no patch) on the same pixels, with the near/far cache produced on the device
    (data_io/cache_helper.py:16-36) checked against the oracle's geometry_guided_near_far."""
    import types
    from neuman_b200 import data as nd
    from neuman_b200.render import SimpleCapture
    from oracle import synth_smpl
    rng = np.random.RandomState(5)
    body = synth_smpl.random_body(seed=1, center=(0.0, 0.0, 2.5))
    H, W = 40, 56
    K = np.array([[70.0, 0, W / 2], [0, 70.0, H / 2], [0, 0, 1]])
    cap = SimpleCapture(K, np.eye(4), H, W, near=0.2, far=6.0)
    cap.near['human'], cap.far['human'] = 0.5, 5.0
    cap.image = rng.randint(0, 256, (H, W, 3)).astype(np.uint8)
    cap.mask = np.zeros((H, W), np.uint8)
    cap.mask[10:30, 18:40] = 1
    cap.binary_mask = cap.mask.copy()
    cap.border_mask = np.zeros((H, W), np.uint8)
    cap.border_mask[8:32, 16:42] = 1
    cap.border_mask[10:30, 18:40] = 0
    cap.frame_id = {'frame_id': 3, 'total_frames': 11}
    nf = nd.near_far_cache_device(cap, body["verts"], body["geo_threshold"])
    # cache vs the oracle on all pixels (grazing rays may flip: ill-conditioned sqrt, as in test_gpu_stages)
    o, d = no.shot_rays(K, np.eye(4), no.all_pixel_coords(H, W))
    near_r, far_r = no.geometry_guided_near_far(torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(body["verts"]),
                                                body["geo_threshold"])
    near_r, far_r = near_r.numpy().reshape(H, W), far_r.numpy().reshape(H, W)
    got = nf.cpu().numpy()
    solid = (near_r < far_r) & ((far_r - near_r) > 1e-3)
    assert solid.sum() > 50 and np.isinf(near_r).sum() > 50
    assert ((got[..., 0] < got[..., 1]) == (near_r < far_r))[solid | np.isinf(near_r)].all()
    # fp32 on the device against the oracle's float64 rays at distance ~2.5: a few 1e-5
    assert np.abs(got[..., 0][solid] - near_r[solid]).max() < 1e-4 and np.abs(got[..., 1][solid] - far_r[solid]).max() < 1e-4
    opt = types.SimpleNamespace(rays_per_batch=300, penalize_lpips=0, dilation=5, body_rays_ratio=0.6, border_rays_ratio=0.1,
                                bkg_rays_ratio=0.3)
    b = nd.HumanRayBatcher(opt, [cap], [nf])
    assert b.get_num_rays_dict(300) == {'num_body_rays': 180, 'num_border_rays': 30, 'num_bkg_rays': 90}
    coords = dict(b.sample_coords(0, need_patch=False))
    c = {k: v.cpu().numpy() for k, v in coords.items()}
    assert (cap.mask[c['num_body_rays'][:, 1], c['num_body_rays'][:, 0]] != 0).all()
    assert (cap.border_mask[c['num_border_rays'][:, 1], c['num_border_rays'][:, 0]] == 1).all()
    assert (cap.mask[c['num_bkg_rays'][:, 1], c['num_bkg_rays'][:, 0]] == 0).all()
    out = b.batch_from_coords(0, coords)
    cache = got.astype(np.float64)
    ref = {k: [] for k in ('color', 'human_near', 'human_far', 'bkg_near', 'bkg_far', 'is_bkg', 'is_hit')}
    for key in b.KEYS:
        cc = c[key]
        num = cc.shape[0]
        ref['color'].append((cap.image[cc[:, 1], cc[:, 0]] / 255).astype(np.float32))
        ref['is_bkg'].append(1 - cap.binary_mask[cc[:, 1], cc[:, 0]])
        ch = cache[cc[:, 1], cc[:, 0]]
        valid = ch[..., 0] < ch[..., 1]
        hn, hf = np.stack([[cap.near['human']]] * num), np.stack([[cap.far['human']]] * num)
        hn[valid, 0] = ch[valid][:, 0]
        hf[valid, 0] = ch[valid][:, 1]
        ref['human_near'].append(hn.astype(np.float32))
        ref['human_far'].append(hf.astype(np.float32))
        ref['bkg_near'].append(np.stack([[cap.near['bkg']]] * num).astype(np.float32))
        ref['bkg_far'].append(np.stack([[cap.far['bkg']]] * num).astype(np.float32))
        ref['is_hit'].append(valid.astype(np.uint8))
    for k, v in ref.items():
        r, g = np.concatenate(v), out[k].cpu().numpy()
        assert g.shape == r.shape, (k, g.shape, r.shape)
        assert np.array_equal(g, r.astype(g.dtype)), k
    assert out['is_bkg'].dtype == torch.long and out['is_hit'].dtype == torch.long and out['origin'].shape == (300, 3)
    assert out['cur_view'] == 3 and abs(out['cur_view_f'] - 3 / 11) < 1e-12 and out['cap_id'] == 0


def _golden_caps(g, prefix, n):
    """SimpleCaptures rebuilt from the arrays tools/make_golden_batches.py stored next to the reference's batches."""
    from neuman_b200.render import SimpleCapture
    caps = []
    for i in range(n):
        p = f"{prefix}{i}_"
        H, W = g[p + "image"].shape[:2]
        nf = g[p + "near_far"]
        cap = SimpleCapture(g[p + "K"], g[p + "c2w"], H, W, near=float(nf[0]), far=float(nf[1]))
        cap.near['human'], cap.far['human'] = float(nf[2]), float(nf[3])
        cap.image, cap.mask, cap.binary_mask = g[p + "image"], g[p + "mask"], g[p + "binary_mask"]
        cap.depth_map, cap.fused_depth_map = g[p + "depth_map"], g[p + "fused_depth_map"]
        if p + "border_mask" in g:
            cap.border_mask = g[p + "border_mask"]
        cap.frame_id = {'frame_id': int(g[p + "frame"][0]), 'total_frames': int(g[p + "frame"][1])}
        caps.append(cap)
    return caps


def _same_batch(out, g, tag, ray_tol=2e-6):
    for key in [k[len(tag) + 5:] for k in g if k.startswith(tag + "_out_")]:
        want, got = g[f"{tag}_out_{key}"], out[key]
        got = got.cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
        assert got.shape == want.shape, (tag, key, got.shape, want.shape)
        if key in ('origin', 'direction'):
            assert np.abs(got - want).max() < ray_tol, (tag, key)
        elif want.dtype.kind == 'f':
            assert np.array_equal(got.astype(want.dtype), want), (tag, key)
        else:
            assert np.array_equal(got.astype(np.int64), want.astype(np.int64)), (tag, key)
            if isinstance(out[key], torch.Tensor) and want.ndim:
                assert out[key].dtype == torch.long, (tag, key)


def test_background_batches_equal_the_reference_dataset():
    """neuman_b200.data.BackgroundRayBatcher on the pixels the UNMODIFIED BackgroundRayDataset.__getitem__
    (datasets/background_rays.py:41-139) drew, against the batch it returned (tests/golden/batches.npz,
    tools/make_golden_batches.py): plain, fused depth, NeRF-T ablation sampling."""
    import types
    from neuman_b200 import data as nd
    g = util.golden("batches.npz")
    caps = _golden_caps(g, "bg_cap", 3)
    for tag, fused, nerft in (("bg", False, False), ("bgf", True, False), ("bgt", False, True)):
        opt = types.SimpleNamespace(rays_per_batch=500, use_fused_depth=fused, ablate_nerft=nerft)
        b = nd.BackgroundRayBatcher(opt, caps)
        bins, xy = g[tag + "_bins"], g[tag + "_coords"]
        coords, at = [], 0
        for n in bins:
            coords.append(None if n == 0 else torch.from_numpy(np.ascontiguousarray(xy[at:at + n], dtype=np.int32)).cuda())
            at += int(n)
        _same_batch(b.batch_from_coords(coords), g, tag)
        # the random part draws from the same admissible sets as the reference did
        if not nerft:
            for cap, c in zip(caps, b.sample_coords()):
                if c is not None:
                    c = c.cpu().numpy()
                    bad = cap.mask[c[:, 1], c[:, 0]] != 0
                    if hasattr(cap, 'border_mask'):
                        bad |= cap.border_mask[c[:, 1], c[:, 0]] != 0
                    assert not bad.any()


def test_human_batches_equal_the_reference_dataset():
    """neuman_b200.data.HumanRayBatcher against the UNMODIFIED HumanRayDataset.__getitem__ (datasets/human_rays.py:100-247)
    on the same pixels and the same near/far cache: no patch (penalize_lpips = 0), patch taken, patch branch enabled but the
    coin of :122 falling on a plain split.  Then the device near/far cache against the reference's
    (data_io/cache_helper.py:16-36) and the shape of a freshly sampled patch."""
    import types
    from neuman_b200 import data as nd
    g = util.golden("batches.npz")
    caps = _golden_caps(g, "hu_cap", 2)
    cache = [g["hu_cap0_cache"], g["hu_cap1_cache"]]
    for tag, lp in (("hu", 0.0), ("hup", 0.1), ("hun", 0.1)):
        opt = types.SimpleNamespace(rays_per_batch=1400, penalize_lpips=lp, dilation=5, body_rays_ratio=0.6,
                                    border_rays_ratio=0.1, bkg_rays_ratio=0.3)
        b = nd.HumanRayBatcher(opt, caps, cache)
        segs = b.plan(need_patch=(tag == "hup"))
        assert [n for _, n in segs] == [int(n) for n in g[tag + "_seg"]], (tag, segs)
        xy, at, coords = g[tag + "_coords"], 0, []
        for key, n in segs:
            coords.append((key, torch.from_numpy(np.ascontiguousarray(xy[at:at + n], dtype=np.int32)).cuda()))
            at += n
        out = b.batch_from_coords(int(g[tag + "_cap"]), coords)
        _same_batch(out, g, tag)
        assert int(out['patch_counter']) == int(g[tag + "_out_patch_counter"])
    # the reference's patch is what patch_coords builds around the same corner
    b = nd.HumanRayBatcher(types.SimpleNamespace(rays_per_batch=1400, penalize_lpips=0.1, dilation=5, body_rays_ratio=0.6,
                                                 border_rays_ratio=0.1, bkg_rays_ratio=0.3), caps, cache)
    ref_patch = g["hup_coords"][:1024]
    centre = (int(ref_patch[0, 0]) + 16, int(ref_patch[0, 1]) + 16)
    assert np.array_equal(b.patch_coords(1, centre).cpu().numpy(), ref_patch)
    for need in (True, False):
        segs = b.sample_coords(1, need_patch=need)
        assert sum(x.shape[0] for _, x in segs) == 1400 and (segs[0][0] == 'num_patch_rays') == need
        if need:
            p = segs[0][1].cpu().numpy().reshape(32, 32, 2)
            H, W = caps[1].image.shape[:2]
            assert (np.diff(p[..., 0], axis=1) == 1).all() and (np.diff(p[..., 1], axis=0) == 1).all()
            assert p.min() >= 0 and p[..., 0].max() < W and p[..., 1].max() < H
    assert nd.get_left_upper_corner(56, 64, (2, 55)) == (0, 24) and nd.get_left_upper_corner(56, 64, (63, 3)) == (32, 0)
    # device near/far cache of the same captures against the reference's cache (float32 rays at distance ~1.5)
    from oracle import synth_smpl
    body = synth_smpl.random_body(seed=1, center=(0.1, -0.05, -0.2))
    for cap, want in zip(caps, cache):
        got = nd.near_far_cache_device(cap, body["verts"], body["geo_threshold"]).cpu().numpy()
        solid = (want[..., 0] < want[..., 1]) & ((want[..., 1] - want[..., 0]) > 1e-3)
        miss = np.isinf(want[..., 0])
        assert solid.sum() > 100 and ((got[..., 0] < got[..., 1]) == (want[..., 0] < want[..., 1]))[solid | miss].all()
        assert np.abs(got[solid] - want[solid]).max() < 1e-4


def test_training_empty_and_scale_and_additivity():
    """Size-independent properties of the training path at a size the oracle cannot reach:
    empty batch; loss-scale invariance (gradients of c*L are c times the gradients of L for c over eight decades:
    the power-of-two loss scale adapts on the device); additivity over the batch (gradients of a 300k-sample
    batch = sum of the gradients of its two halves: persistent-kernel rounds, TMA tails and the split-K
    reduction of k_dw_gemm agree)."""
    from tests.util import product_nets
    coarse, _, _ = product_nets(DEV)
    j = coarse

    def grads(pts, views, g):
        j.zero_grad()
        (j(pts, views) * g).sum().backward()
        return {k: p.grad.detach().clone() for k, p in j.nerf.named_parameters()}
    # empty
    e = torch.zeros(0, 3, device=DEV)
    raw = j(e, e)
    assert raw.shape == (0, 4)
    raw.sum().backward()
    assert all(p.grad is not None and float(p.grad.abs().max()) == 0.0 for p in j.nerf.parameters())
    # loss-scale invariance
    torch.manual_seed(3)
    n = 5000
    pts = torch.randn(n, 3, device=DEV)
    views = torch.nn.functional.normalize(torch.randn(n, 3, device=DEV), dim=-1)
    g = torch.randn(n, 4, device=DEV)
    base = grads(pts, views, g)
    for c in (1e-4, 1e4):
        sc = grads(pts, views, g * c)
        for k in base:
            assert torch.isfinite(sc[k]).all()
            assert _rel(sc[k] / c, base[k]) < 3e-3, (c, k, _rel(sc[k] / c, base[k]))    # fp16 rounding at different mantissas
    # additivity at scale (several persistent rounds per kernel)
    n = 300000 + 77
    pts = torch.randn(n, 3, device=DEV)
    views = torch.nn.functional.normalize(torch.randn(n, 3, device=DEV), dim=-1)
    g = torch.randn(n, 4, device=DEV) * (torch.rand(n, 1, device=DEV) < 0.5)      # half of the rows carry no gradient
    h = n // 2 + 13
    full = grads(pts, views, g)
    a = grads(pts[:h], views[:h], g[:h])
    b = grads(pts[h:], views[h:], g[h:])
    for k in full:
        assert _rel(a[k] + b[k], full[k]) < 2e-3, (k, _rel(a[k] + b[k], full[k]))
