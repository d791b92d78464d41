"""NeRF-T nets (the reference's --ablate_nerft background nets: position input (x, y, z, t)) on the GPU: both forward
kernels against the reference goldens (tests/golden/nerft.npz), ragged sizes, render_vanilla(ablate_nerft=True) with chunk
and pixel-list invariance, the training forward and backward in their exact windows, parameter gradients, the loss_func
step with per-ray times, the entry points that refuse NeRF-T slots, slot kind switching and the drop-in."""
import copy

import numpy as np
import pytest
import torch

import neuman_b200 as nb
from neuman_b200 import _lib, autograd, ops, render
from oracle import neuman_oracle as no
from oracle import scenes
from tests import nerft_cases as nc
from tests import tc_exact as tx
from tests import util

pytestmark = pytest.mark.gpu
DEV = "cuda"
MODES = {"simt": _lib.NM_MLP_SIMT_F32, "tc": _lib.NM_MLP_TC_F16}
RAW_TOL = {"simt": 2e-5, "tc": 1e-3}
TOL = 1e-4
UNSUPPORTED = -3          # NM_ERR_UNSUPPORTED


@pytest.fixture(autouse=True)
def clear_range_flag():
    """The range flag is sticky per context: tests elsewhere in the suite saturate it on purpose.  Start each test clean
    (the renderers with host output raise on a set flag)."""
    ctx = ops._ctx_for(torch.zeros(1, device=DEV))
    ctx.lib.nm_range_status(ctx.h, 1, ctx.stream())                 # NM_ERR_RANGE here belongs to an earlier test
    yield


@pytest.fixture(scope="module")
def gold():
    return util.golden("nerft.npz")


@pytest.fixture(scope="module")
def nets():
    return tuple(j.to(DEV) for j in nc.nerft_nets(nb.build_nerf, nb.default_opt))


def _cap(frame):
    f = util.golden("frames.npz")
    cap = nb.SimpleCapture(np.asarray(f["van_K"]), np.asarray(f["van_c2w"]).astype(np.float64), nc.VAN["H"], nc.VAN["W"],
                           nc.NEAR, nc.FAR)
    cap.frame_id = {"frame_id": nc.FRAMES[frame][0], "total_frames": nc.FRAMES[frame][1]}
    return cap


# ---- 1. forward -------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["simt", "tc"])
def test_forward_against_reference_goldens(gold, nets, mode):
    pts, views = torch.from_numpy(gold["pts"]).to(DEV), torch.from_numpy(gold["views"]).to(DEV)
    for name, j in zip(("coarse", "fine"), nets):
        y = ops.joiner_forward(j, pts, views, mode=MODES[mode]).cpu().numpy()
        assert np.abs(y - gold[f"net_{name}"]).max() < RAW_TOL[mode], (mode, name)
        # the same points at two times: the kernel's raw differs as the reference's does
        a, b = y[300:350], y[350:400]
        ga, gb = gold[f"net_{name}"][300:350], gold[f"net_{name}"][350:400]
        assert np.abs((a - b) - (ga - gb)).max() < 2 * RAW_TOL[mode] and np.abs(a - b).max() > 1e-2


def test_ragged_sizes_and_kernel_agreement(nets):
    """Every sample is computed independently of its tile: the first n rows of a 70 000-sample call are bit-equal to an
    n-sample call (n = 1, 127, 128, 129: partial and full tiles); the tensor-core kernel against the fp32 kernel."""
    g = torch.Generator().manual_seed(21)
    n = 70000
    pts = torch.cat([torch.randn(n, 3, generator=g) * 0.8, torch.rand(n, 1, generator=g)], 1).to(DEV)
    views = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).to(DEV)
    full = ops.joiner_forward(nets[0], pts, views, mode=MODES["tc"])
    for m in (1, 127, 128, 129):
        assert torch.equal(ops.joiner_forward(nets[0], pts[:m], views[:m], mode=MODES["tc"]), full[:m]), m
    ref = ops.joiner_forward(nets[0], pts, views, mode=MODES["simt"])
    assert (full - ref).abs().max() < RAW_TOL["tc"]


# ---- 2. render_vanilla(ablate_nerft=True) ------------------------------------------------------
@pytest.mark.parametrize("mode", ["simt", "tc"])
def test_render_vanilla_nerft_against_reference(gold, nets, mode, monkeypatch):
    monkeypatch.setenv("NEUMAN_MLP_MODE", mode)
    c, fn = nets
    H, W, S, N = nc.VAN["H"], nc.VAN["W"], nc.VAN["S"], nc.VAN["N"]
    for i in (0, 1):
        cap = _cap(i)
        t = nc.frame_time(*nc.FRAMES[i])
        rgb, dep = render.render_vanilla_range(c, cap, fn, S, N, pix0=0, n=H * W, host_out=False, frame_time=t)
        b_rgb, b_dep = render.render_vanilla_range(c, cap, fn, S, N, pix0=0, n=H * W, host_out=False, chunk=777, frame_time=t)
        assert torch.equal(rgb, b_rgb) and torch.equal(dep, b_dep)                       # chunk-invariant
        pix = torch.arange(H * W - 1, -1, -3, device=DEV, dtype=torch.int32)
        p_rgb, p_dep = render.render_vanilla_range(c, cap, fn, S, N, pixels=pix, host_out=False, frame_time=t)
        assert torch.equal(p_rgb, rgb[pix.long()]) and torch.equal(p_dep, dep[pix.long()])   # pixel list = range
        e_rgb = np.abs(rgb.cpu().numpy() - gold[f"van{i}_rgb"].reshape(-1, 3)).max()
        e_dep = np.abs(dep.cpu().numpy() - gold[f"van{i}_depth"].reshape(-1))
        gate = max(1e-4, 1.5 * float(gold[f"van{i}_floor16_depth"].max())) if mode == "tc" else 1e-4
        assert e_rgb < TOL and (e_dep <= gate).all(), (i, e_rgb, float(e_dep.max()))
        # the reference's signature: host numpy arrays of the whole frame
        r2, d2 = nb.render_vanilla(c, cap, fine_net=fn, samples_per_ray=S, importance_samples_per_ray=N, return_depth=True,
                                   ablate_nerft=True)
        assert np.array_equal(r2.reshape(-1, 3), rgb.cpu().numpy()) and np.array_equal(d2.reshape(-1), dep.cpu().numpy())


def test_samplers_append_the_time_column(nets):
    R, S = 64, 16
    g = torch.Generator().manual_seed(3)
    rb = {"origin": torch.randn(R, 3, generator=g).to(DEV),
          "direction": torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1).to(DEV),
          "near": torch.zeros(R, 1, device=DEV), "far": torch.full((R, 1), 3.0, device=DEV)}
    t = torch.ones(R, S, 1, device=DEV) * (7 / 30)
    p0, d0, z0 = ops.ray_to_samples(rb, S)
    p, d, z = ops.ray_to_samples(rb, S, append_t=t)
    assert p.shape == (R, S, 4) and torch.equal(p[..., :3], p0) and torch.equal(p[..., 3:], t)
    assert torch.equal(d, d0) and torch.equal(z, z0)
    w = torch.rand(R, S, generator=g).to(DEV)
    tf = torch.ones(R, S + 8, 1, device=DEV) * 0.25
    q0, _, _ = ops.ray_to_importance_samples(rb, z, w, 8)
    q, _, _ = ops.ray_to_importance_samples(rb, z, w, 8, append_t=tf)
    assert q.shape == (R, S + 8, 4) and torch.equal(q[..., :3], q0) and torch.equal(q[..., 3:], tf)


# ---- 3. entry points that refuse NeRF-T slots ---------------------------------------------------
def test_drivers_without_time_refuse_nerft_slots(nets):
    c, fn = nets
    cap = _cap(0)
    H, W = nc.VAN["H"], nc.VAN["W"]
    with pytest.raises(_lib.NmError, match="-3"):
        render.render_vanilla_range(c, cap, fn, 8, 8, pix0=0, n=H * W, host_out=False)
    plain, _ = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False), 8)
    plain = plain.to(DEV)
    with pytest.raises(_lib.NmError, match="-3"):                    # the time driver needs NeRF-T nets
        render.render_vanilla_range(plain, cap, None, 8, 8, pix0=0, n=H * W, host_out=False, frame_time=0.5)
    z = torch.linspace(0, 1, 8, device=DEV).repeat(4, 1)
    o, d = torch.zeros(4, 3, device=DEV), torch.ones(4, 3, device=DEV)
    with pytest.raises(_lib.NmError, match="-3"):
        ops.mlp_forward_rays(c, o, d, z)
    ctx = ops._ctx_for(z)
    slot = ops.net_slot(c, ctx)
    buf = torch.zeros(1 << 16, device=DEV)
    p = ops._p(buf)
    assert ctx.lib.nm_pe_backward(ctx.h, slot, 0, p, 0, p, 96, None, 4, p, ctx.stream()) == UNSUPPORTED    # no input gradient
    assert ops.joiner_forward(plain, torch.zeros(4, 3, device=DEV), torch.ones(4, 3, device=DEV)).shape == (4, 4)


# ---- 4. slot kind switching -------------------------------------------------------------------
def test_slot_switches_kind(nets):
    """One slot packed view -> NeRF-T -> view: each forward equals that of a fresh slot."""
    ctx = ops._ctx_for(torch.zeros(1, device=DEV))
    view, _ = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False), 8)
    view, nt = view.to(DEV), nets[0]
    g = torch.Generator().manual_seed(4)
    pts = torch.cat([torch.randn(2000, 3, generator=g), torch.rand(2000, 1, generator=g)], 1).to(DEV)
    views = torch.nn.functional.normalize(torch.randn(2000, 3, generator=g), dim=-1).to(DEV)

    def run(j, mode):
        return ops.joiner_forward(j, pts if ops.is_nerft(j) else pts[:, :3].contiguous(), views, mode=MODES[mode])
    fresh = {(id(j), m): run(j, m) for j in (view, nt) for m in MODES}
    saved = (dict(ctx.slots), list(ctx.slot_keys), list(ctx.slot_used))
    try:
        for j in (view, nt, view, nt):
            ops.invalidate_net(j)
            ctx.slots = {}
            ctx.slot_keys = [None] + [("held",)] * (len(ctx.slot_keys) - 1)    # the only free slot: 0
            assert ops.net_slot(j, ctx) == 0
            for m in MODES:
                assert torch.equal(run(j, m), fresh[(id(j), m)]), m
    finally:
        slots, keys, used = saved
        ctx.slots = {k: v for k, v in slots.items() if v != 0}
        ctx.slot_keys = [None if i == 0 else k for i, k in enumerate(keys)]
        ctx.slot_used = used
        for j in (view, nt):
            ops.invalidate_net(j)


# ---- 5. drop-in -------------------------------------------------------------------------------
def test_dropin_runs_nerft_calls_on_the_library(gold):
    """Under install() the stand-in reference's render_vanilla(ablate_nerft=True) and Joiner.forward on (x, y, z, t) run on
    the library: the reference functions are wrapped in spies before install() stashes them, and the spies are never
    called; the results match the reference goldens."""
    from tests.standin_reference import standin
    with standin() as r:
        calls = []
        orig = r.render_utils.render_vanilla

        def spy(*a, **k):
            calls.append("render_vanilla")
            return orig(*a, **k)
        r.render_utils.render_vanilla = spy
        nb.install()
        try:
            c, fn = (j.to(DEV) for j in nc.nerft_nets(r.vanilla.build_nerf, nb.default_opt))
            assert type(c).__module__ == "models.vanilla" and nb.dropin.supported_joiner(c)
            H, W, S, N = nc.VAN["H"], nc.VAN["W"], nc.VAN["S"], nc.VAN["N"]
            l0 = ops.Context.get(0).launch_count()
            with torch.no_grad():
                rgb = r.render_utils.render_vanilla(c, _cap(1), fine_net=fn, rays_per_batch=100, samples_per_ray=S,
                                                    importance_samples_per_ray=N, ablate_nerft=True)
                raw = c(torch.from_numpy(gold["pts"]).to(DEV), torch.from_numpy(gold["views"]).to(DEV))
            assert ops.Context.get(0).launch_count() > l0 and raw.is_cuda
            assert np.abs(rgb - gold["van1_rgb"]).max() < TOL
            assert np.abs(raw.cpu().numpy() - gold["net_coarse"]).max() < RAW_TOL["tc"]
            assert calls == [], calls                                  # the reference function was never reached
        finally:
            nb.dropin.uninstall()


# ---- 6. training: forward stash and backward planes in their exact windows ----------------------
def _inputs4(n, seed):
    g = torch.Generator().manual_seed(seed)
    pts = torch.cat([torch.randn(n, 3, generator=g) * 0.8, torch.rand(n, 1, generator=g)], 1)
    views = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    return pts.to(DEV), views.to(DEV)


def _forward_train(net, pts, views):
    ctx = ops._ctx_for(pts)
    slot = ops.net_slot(net, ctx)
    n = pts.shape[0]
    h = dict(device=DEV, dtype=torch.float16)
    sx, sf, sv = torch.empty(8, n, 256, **h), torch.empty(n, 256, **h), torch.empty(n, 128, **h)
    sm = torch.empty(9, n, 8, device=DEV, dtype=torch.int32)
    raw = torch.empty(n, 4, device=DEV)
    ctx.check(ctx.lib.nm_mlp_forward_train(ctx.h, slot, ops._p(pts), ops._p(views), n, 0, ops._p(raw), ops._p(sx), ops._p(sf),
                                           ops._p(sv), ops._p(sm), ctx.stream()))
    return sx, sf, sv, sm, raw


def _plane96(net, pts):
    ctx = ops._ctx_for(pts)
    pe = torch.empty(pts.shape[0], 96, device=DEV, dtype=torch.float16)
    ctx.check(ctx.lib.nm_encode_f16(ctx.h, ops.net_slot(net, ctx), 0, ops._p(pts), 0, pts.shape[0], ops._p(pe), ctx.stream()))
    return pe


@pytest.mark.parametrize("n", [129, 20000])
def test_training_forward_in_exact_windows(nets, n):
    """Layers 0..7 of the training stash inside their exact windows over the kernel's K order (the time slab included),
    computed from the [n,96] encoding plane; its sign words; the training raw equals the inference raw."""
    net = nets[0]
    pts, views = _inputs4(n, 7)
    sx, sf, sv, sm, raw = _forward_train(net, pts, views)
    assert torch.equal(raw, ops.joiner_forward(net, pts, views, mode=MODES["tc"]))
    pe96 = _plane96(net, pts).double()
    assert torch.equal(pe96[:, 84], torch.ones_like(pe96[:, 84])) and not pe96[:, 85:].any()
    # the plane in the reference's column order: x, y, z, t exactly rounded, sin/cos channels within the encoder's error
    ref = no.embed(pts.cpu(), util.oracle_params(copy.deepcopy(net).cpu()).pos_pe).double().to(DEV)
    assert torch.equal(pe96[:, :4], tx.r16(pts.double()))
    assert (pe96[:, 4:84] - ref[:, 4:]).abs().max() < 1e-3
    W16, _ = tx.weights(net, DEV)
    pc = nc.kernel_pos_columns()
    sxd = sx.double()
    for l in range(8):
        if l in (0, 5):
            blocks = nc.nerft_blocks(W16, l, pe96, sxd)
        else:
            w, b = W16[f'pts_linears.{l}.weight'], W16[f'pts_linears.{l}.bias']
            wb = torch.zeros(b.shape[0], 16, dtype=torch.float64, device=DEV)
            wb[:, 15] = b
            blocks = [(sxd[l - 1], w), (pe96[:, pc][:, 48:64], wb)]
        c = tx.check16(f"layer{l}", sx[l], *tx.mma_ref(blocks), relu=True)
        assert c.n_bad == 0, c.message()
        assert torch.equal(sm[l].to(torch.int64) & 0xFFFFFFFF, tx.sign_words(sx[l]) & 0xFFFFFFFF), ("sign words", l)


def test_backward_planes_in_exact_windows(nets):
    """Every element of g_v, g_f and g_pre[7..0] inside its exact window on the kernel's own planes (layer 5's hidden
    columns start at 84 in a NeRF-T net)."""
    net = nets[1]
    n = 20000
    pts, views = _inputs4(n, 21)
    sx, sf, sv, sm, _ = _forward_train(net, pts, views)
    g = torch.randn(n, 4, device=DEV, generator=torch.Generator(DEV).manual_seed(3))
    scale = autograd._pow2_scale(g, 256.0)
    ctx = ops._ctx_for(pts)
    h = dict(device=DEV, dtype=torch.float16)
    g_pre, g_f, g_v = torch.empty(8, n, 256, **h), torch.empty(n, 256, **h), torch.empty(n, 128, **h)
    ctx.check(ctx.lib.nm_mlp_backward(ctx.h, ops.net_slot(net, ctx), ops._p(g), ops._p(scale), n, ops._p(sv), ops._p(sm),
                                      ops._p(g_pre), ops._p(g_f), ops._p(g_v), ctx.stream()))
    W16, W32 = tx.weights(net, DEV)
    for c in tx.backward_checks(W16, W32, scale, g, sx, sv, g_pre, g_f, g_v):
        assert c.n_bad == 0, c.message()


# ---- 7. parameter gradients ----------------------------------------------------------------------
def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def test_parameter_gradients(nets, monkeypatch):
    """Gradients of every parameter against the torch restatement of the two kernel launches on the same stash (2e-3),
    fp32 autograd through the oracle with fp16-rounded operands (3e-2) and plain fp32 autograd (8e-2)."""
    net = copy.deepcopy(nets[0])
    n = 3000
    pts, views = _inputs4(n, 11)
    g = torch.randn(n, 4, device=DEV, generator=torch.Generator(DEV).manual_seed(5))

    def product(torch_chain):
        if torch_chain:
            monkeypatch.setattr(autograd, "_chain_kernel", util.chain_torch)
            monkeypatch.setattr(autograd, "_dw_kernel", util.dw_torch)
        for p in net.parameters():
            p.grad = None
        autograd.joiner_forward(net, pts, views).backward(g)
        monkeypatch.undo()
        return {k: p.grad.clone() for k, p in net.nerf.named_parameters()}
    got = product(False)
    chain = product(True)
    assert set(got) == {k for k, _ in net.nerf.named_parameters()}
    for k in got:
        assert torch.isfinite(got[k]).all(), k
        assert _rel(got[k], chain[k]) < 2e-3, ("kernel vs torch chain", k, _rel(got[k], chain[k]))
    for operands, tol in (("f16", 3e-2), (None, 8e-2)):
        P = util.oracle_params(copy.deepcopy(net).to("cpu"))
        for k in P.sd:
            P.sd[k].requires_grad_(True)
        with no.precision(operands=operands):
            no.net_forward(P, pts.cpu(), views.cpu()).backward(g.cpu())
        for k in got:
            ref = P.sd["nerf." + k].grad
            assert _rel(got[k].cpu(), ref) < tol, (operands, k, _rel(got[k].cpu(), ref))


# ---- 8. the background trainer's step with per-ray times ----------------------------------------
def test_loss_func_with_viewf_list_matches_autograd(nets):
    """train.vanilla_loss_func(opt.ablate_nerft) on a batch whose rays come from 4 frames (viewf_list): losses and every
    parameter gradient against CPU autograd of the oracle on the same samples; then a few Adam steps lower the loss."""
    from neuman_b200 import train as nt
    coarse, fine = (copy.deepcopy(j) for j in nets)
    S, N = 32, 32
    opt = nb.default_opt(samples_per_ray=S, importance_samples_per_ray=N, perturb=1.0, raw_noise_std=1.0, margin=0.9,
                         ablate_nerft=True)
    R = 300
    torch.manual_seed(5)
    o = torch.randn(R, 3) * 0.1
    d = torch.nn.functional.normalize(torch.randn(R, 3), dim=-1)
    tv = torch.tensor([nc.frame_time(f, 30) for f in (0, 7, 19, 29)]).repeat_interleave(R // 4)[:, None]
    batch = dict(origin=o.to(DEV), direction=d.to(DEV), near=torch.full((R,), 0.5, device=DEV),
                 far=torch.full((R,), 4.0, device=DEV), color=torch.rand(R, 3, device=DEV),
                 depth=(1.5 + torch.rand(R)).to(DEV), viewf_list=tv.to(DEV))
    t_rand = torch.rand(R, S)
    noise = (torch.randn(R, S), torch.randn(R, S + N))
    kw = dict(check_bad_weights=False, penalize_empty_space=0.1, t_rand=t_rand.to(DEV), noise=tuple(x.to(DEV) for x in noise))
    losses = nt.vanilla_loss_func(coarse, fine, batch, opt, **kw)
    sum(losses).backward()
    with torch.no_grad():
        _, _, z = nb.ray_to_samples(batch, S, perturb=1.0, t_rand=t_rand.to(DEV))
        pc = nb.ray_to_samples(batch, S, perturb=1.0, t_rand=t_rand.to(DEV), append_t=tv.to(DEV).repeat(1, S)[..., None])[0]
        w = nb.raw2outputs(coarse(pc, batch['direction'][:, None].expand(R, S, 3)), z, batch['direction'], raw_noise_std=1.0,
                           white_bkg=True, noise=noise[0].to(DEV))[3]
        _, _, Fz = nb.ray_to_importance_samples(batch, z, w, N)
    z, Fz = z.cpu(), Fz.cpu()
    onets = [util.oracle_params(copy.deepcopy(coarse).cpu()), util.oracle_params(copy.deepcopy(fine).cpu())]
    for net in onets:
        for k in net.sd:
            net.sd[k].requires_grad_(True)
    import torch.nn.functional as F

    def side(net, zz, nz):
        pts = o[:, None, :] + d[:, None, :] * zz[..., None]
        pts = torch.cat([pts, tv.repeat(1, zz.shape[1])[..., None]], -1)
        raw = no.net_forward(net, pts, d[:, None, :].expand(R, zz.shape[1], 3))
        rgb = no.raw2outputs(raw, zz, d, raw_noise_std=1.0, white_bkg=True, noise=nz)[0]
        m = zz < (batch['depth'].cpu()[:, None] * 0.9)
        s = raw[m][:, 3]
        return F.mse_loss(rgb, batch['color'].cpu()), F.l1_loss(torch.tanh(torch.relu(s)), torch.zeros_like(s)) * 0.1
    ref = side(onets[0], z, noise[0]) + side(onets[1], Fz, noise[1])
    sum(ref).backward()
    for a, b in zip(losses, ref):
        assert abs(float(a) - float(b)) < 2e-4 * max(1.0, abs(float(b))), (float(a), float(b))
    for j, net in ((coarse, onets[0]), (fine, onets[1])):
        for k, p in j.nerf.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all(), k
            assert _rel(p.grad.cpu(), net.sd["nerf." + k].grad) < 8e-2, (k, _rel(p.grad.cpu(), net.sd["nerf." + k].grad))
    optim = torch.optim.Adam(list(coarse.parameters()) + list(fine.parameters()), lr=5e-4)
    first = last = None
    for it in range(6):
        last = float(nt.train_batch(coarse, fine, optim, batch, opt, iteration=it, **kw))
        first = last if first is None else first
    assert np.isfinite(last) and last < first, (first, last)


def test_dropin_trains_nerft_nets_on_the_library(gold):
    """Under install(train=True), Joiner.forward of a NeRF-T net under autograd runs the library's training kernels (the
    stand-in reference's own forward is never reached) and its gradients equal those of autograd.joiner_forward."""
    from tests.standin_reference import standin
    with standin() as r:
        calls = []
        ref_fwd = r.vanilla.Joiner.forward

        def spy(self, *a, **k):
            calls.append("forward")
            return ref_fwd(self, *a, **k)
        r.vanilla.Joiner.forward = spy
        nb.install(train=True)
        try:
            c, _ = nc.nerft_nets(r.vanilla.build_nerf, nb.default_opt)
            c = c.to(DEV)
            pts, views = torch.from_numpy(gold["pts"]).to(DEV), torch.from_numpy(gold["views"]).to(DEV)
            l0 = ops.Context.get(0).launch_count()
            c(pts, views).sum().backward()
            assert ops.Context.get(0).launch_count() > l0 and calls == [], calls
            got = {k: p.grad.clone() for k, p in c.nerf.named_parameters()}
            for p in c.parameters():
                p.grad = None
            autograd.joiner_forward(c, pts, views).sum().backward()
            for k, p in c.nerf.named_parameters():
                assert torch.equal(got[k], p.grad) or _rel(got[k], p.grad) < 1e-5, k
        finally:
            nb.dropin.uninstall()
            r.vanilla.Joiner.forward = ref_fwd
