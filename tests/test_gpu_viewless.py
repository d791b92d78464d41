"""View-independent nets (NeRF with use_viewdirs=False: one output_linear [4,256] on layer 7, no direction input; the
reference's --use_viewdirs False / --specular_can False) on the GPU: forward kernels against the oracle, exact windows
of the training forward, the backward chain and gradients, the frame drivers with any mix of net kinds, slot kind
switching, the range guard and the drop-in."""
import copy

import numpy as np
import pytest
import torch

import neuman_b200 as nb
from neuman_b200 import _lib, autograd, ops, render
from oracle import neuman_oracle as no
from oracle import scenes
from oracle import synth_smpl
from tests import tc_exact as tx
from tests import util
from tests import viewless_cases as vc
from tests.viewless_cases import head_check

pytestmark = pytest.mark.gpu
DEV = "cuda"
MODES = {"simt": _lib.NM_MLP_SIMT_F32, "tc": _lib.NM_MLP_TC_F16}
RAW_TOL = {"simt": 2e-5, "tc": 1e-3}
TOL = 1e-4


def viewless_net(posenc, seed, boost=True):
    """A seeded use_viewdirs=False Joiner; the output bias is raised so that renders are not empty."""
    coarse, fine = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False, use_viewdirs=False, posenc=posenc), seed)
    if boost:
        with torch.no_grad():
            for j in (coarse, fine):
                j.nerf.output_linear.weight[3].mul_(8.0)
                j.nerf.output_linear.bias[3].add_(0.3)
    return coarse, fine


@pytest.fixture(autouse=True)
def clear_range_flag():
    """The range flag is sticky per context: tests elsewhere in the suite saturate it on purpose.  Start each test clean
    (the renderers with host output raise on a set flag)."""
    ctx = ops._ctx_for(torch.zeros(1, device=DEV))
    ctx.lib.nm_range_status(ctx.h, 1, ctx.stream())                 # NM_ERR_RANGE here belongs to an earlier test
    yield


@pytest.fixture(scope="module")
def nets():
    c, f = viewless_net("posenc", 3)
    h, _ = viewless_net("rotate", 4)
    return c.to(DEV), f.to(DEV), h.to(DEV)


def _oracle(net, pts):
    net.to("cpu")
    try:
        with torch.no_grad():
            return no.net_forward(util.oracle_params(net), pts.cpu(), None)
    finally:
        net.to(DEV)


def _inputs(n, seed):
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(n, 3, generator=g) * 0.8
    views = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    return pts, views


# ---- 1. forward -------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["simt", "tc"])
@pytest.mark.parametrize("which", [0, 2])
def test_forward_against_oracle_and_views_ignored(nets, mode, which):
    net = nets[which]
    pts, views = _inputs(5000, which)
    ref = _oracle(net, pts)
    a = ops.joiner_forward(net, pts.to(DEV), views.to(DEV), mode=MODES[mode])
    assert (a.cpu() - ref).abs().max() < RAW_TOL[mode]
    b = ops.joiner_forward(net, pts.to(DEV), -views.to(DEV), mode=MODES[mode])
    c = ops.joiner_forward(net, pts.to(DEV), None, mode=MODES[mode])
    assert torch.equal(a, b) and torch.equal(a, c)                     # raw does not depend on the views
    with torch.no_grad():
        d = net(pts.to(DEV))                                           # models.Joiner.forward without views
    if mode == "tc":
        assert torch.equal(a, d)


@pytest.fixture(scope="module")
def gold():
    return util.golden("viewless.npz")


@pytest.mark.parametrize("mode", ["simt", "tc"])
@pytest.mark.parametrize("pe", ["posenc", "rotate"])
def test_forward_against_reference_goldens(gold, mode, pe):
    s = util.golden("stages.npz")
    pts, views = torch.from_numpy(s["n_pts"]).to(DEV), torch.from_numpy(s["n_views"]).to(DEV)
    for name, j in zip(("coarse", "fine"), vc.viewless_nets(nb.build_nerf, nb.default_opt, pe)):
        assert vc.checksum(j) == gold[f"net_{pe}_{name}_sum"]
        j = j.to(DEV)
        y = ops.joiner_forward(j, pts, views, mode=MODES[mode])
        assert np.abs(y.cpu().numpy() - gold[f"net_{pe}_{name}"]).max() < RAW_TOL[mode], (pe, name)
        assert torch.equal(y, ops.joiner_forward(j, pts, None, mode=MODES[mode]))


@pytest.mark.parametrize("mode", ["simt", "tc"])
def test_rays_mode_equals_pts_mode(nets, mode):
    torch.manual_seed(5)
    R, S = 300, 96
    o, d = torch.randn(R, 3).to(DEV), torch.nn.functional.normalize(torch.randn(R, 3), dim=-1).to(DEV)
    pts, dirs, z = nb.ray_to_samples({"origin": o, "direction": d, "near": torch.zeros(R, 1, device=DEV),
                                      "far": torch.full((R, 1), 3.0, device=DEV)}, S)
    a = ops.mlp_forward_rays(nets[0], o, d, z, mode=MODES[mode])
    b = ops.joiner_forward(nets[0], pts, dirs, mode=MODES[mode])
    assert torch.equal(a, b)


# ---- 2. exact windows of the training forward -------------------------------------------------
PAD = 4096          # sentinel elements after every output buffer
SENT = -12345


def _padded(numel, dtype):
    buf = torch.empty(numel + PAD, device=DEV, dtype=dtype)
    if dtype == torch.float32:
        buf.fill_(float(SENT))
    else:
        buf.view(torch.int16 if dtype == torch.float16 else torch.int32).fill_(SENT)
    return buf


def _intact(buf, numel):
    t = buf[numel:]
    if buf.dtype == torch.float32:
        return bool((t == float(SENT)).all())
    return bool((t.view(torch.int16 if buf.dtype == torch.float16 else torch.int32) == SENT).all())


def _forward_train(net, pts):
    ctx = ops._ctx_for(pts)
    slot = ops.net_slot(net, ctx)
    n = pts.shape[0]
    sx, sm, raw = _padded(8 * n * 256, torch.float16), _padded(8 * n * 8, torch.int32), _padded(n * 4, torch.float32)
    ctx.check(ctx.lib.nm_mlp_forward_train(ctx.h, slot, ops._p(pts), None, n, 0, ops._p(raw), ops._p(sx), None, None,
                                           ops._p(sm), ctx.stream()))
    torch.cuda.synchronize()
    for b, k in ((sx, 8 * n * 256), (sm, 8 * n * 8), (raw, n * 4)):
        assert _intact(b, k), "sentinel after an output buffer overwritten"
    return sx[:8 * n * 256].view(8, n, 256), sm[:8 * n * 8].view(8, n, 8), raw[:n * 4].view(n, 4)


def _T():
    return 128 * torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("which", [0, 2])
@pytest.mark.parametrize("size", ["1", "129", "3T-5"])
def test_training_forward_in_exact_windows(nets, which, size):
    net = nets[which]
    n = {"1": 1, "129": 129, "3T-5": 3 * _T() - 5}[size]
    pts, _ = _inputs(n, 7 + which)
    pts = pts.to(DEV)
    sx, sm, raw = _forward_train(net, pts)
    assert torch.equal(raw, ops.joiner_forward(net, pts, None, mode=MODES["tc"]))     # inference kernel = training raw
    W16, W32 = tx.weights(net, DEV)
    pe = torch.empty(n, 64, device=DEV, dtype=torch.float16)
    ctx = ops._ctx_for(pts)
    ctx.check(ctx.lib.nm_encode_f16(ctx.h, ops.net_slot(net, ctx), 0, ops._p(pts), 0, n, ops._p(pe), ctx.stream()))
    pe = pe.double()
    for l in range(8):
        c = tx.check16(f"layer{l}", sx[l], *tx.mma_ref(tx.hidden_blocks(W16, l, pe, sx.double())), relu=True)
        assert c.n_bad == 0, c.message()
        assert torch.equal(sm[l].to(torch.int64) & 0xFFFFFFFF, tx.sign_words(sx[l]) & 0xFFFFFFFF), ("sign words", l)
    c = head_check(W16, W32, sx[7].double(), raw)
    assert c.n_bad == 0, c.message()


def test_direction_entry_points_are_unsupported(nets):
    ctx = ops._ctx_for(torch.zeros(1, device=DEV))
    slot = ops.net_slot(nets[0], ctx)
    x = torch.zeros(4, 3, device=DEV)
    out = torch.empty(4, 32, device=DEV, dtype=torch.float16)
    assert ctx.lib.nm_encode_f16(ctx.h, slot, 1, ops._p(x), 0, 4, ops._p(out), ctx.stream()) == -3
    d_enc, d_x = torch.zeros(4, 32, device=DEV), torch.empty(4, 3, device=DEV)
    assert ctx.lib.nm_pe_backward(ctx.h, slot, 1, ops._p(x), 0, ops._p(d_enc), 32, None, 4, ops._p(d_x), ctx.stream()) == -3


# ---- 3. backward --------------------------------------------------------------------------------
def chain_torch_viewless(joiner, P, stash, g):
    """k_mlp_tc_bwd_noview restated with torch on the same stash: the K = 4 head, then layers 7..1."""
    from neuman_b200.autograd import _mm32, _pow2_scale
    sx, _, _, _ = stash
    n_pe = joiner.pos_pe.out_dim
    scale = _pow2_scale(g, 256.0)
    gs = g * scale
    dX = gs @ P['output_linear.weight'].detach().float()
    g_pre = torch.empty_like(sx)
    for l in range(7, -1, -1):
        g_pre[l] = (dX * (sx[l] > 0)).half()
        if l > 0:
            w = P['pts_linears.%d.weight' % l].detach().half()
            dX = _mm32(g_pre[l], w[:, n_pe:].contiguous() if l == 5 else w)
    return g_pre, None, None, 1.0 / scale


def dw_torch_viewless(ctx, g_pre, g_f, g_v, sx, sf, n):
    from neuman_b200.autograd import _mm32
    assert g_f is None and g_v is None and sf is None
    dw = torch.zeros(9, 256, 256, device=g_pre.device, dtype=torch.float32)
    db = torch.zeros(9, 256, device=g_pre.device, dtype=torch.float32)
    for k in range(7):
        dw[k] = _mm32(g_pre[k + 1].t(), sx[k])
        db[k] = g_pre[k + 1].float().sum(0)
    return dw, db


@pytest.mark.parametrize("which", [0, 2])
def test_backward_planes_in_exact_windows_and_against_torch_chain(nets, which):
    """Every element of g_pre[7..0] from k_mlp_tc_bwd_noview: inside its exact window computed on the kernel's own plane
    above, and next to the torch restatement of the whole chain on the same stash; sentinels after g_pre untouched."""
    from neuman_b200.autograd import _pow2_scale
    net = nets[which]
    n = 3 * _T() - 5
    pts, _ = _inputs(n, 21 + which)
    pts = pts.to(DEV)
    sx, sm, _ = _forward_train(net, pts)
    g = torch.randn(n, 4, device=DEV, generator=torch.Generator(DEV).manual_seed(which))
    scale = _pow2_scale(g, 256.0)
    ctx = ops._ctx_for(pts)
    gp = _padded(8 * n * 256, torch.float16)
    ctx.check(ctx.lib.nm_mlp_backward(ctx.h, ops.net_slot(net, ctx), ops._p(g), ops._p(scale), n, None, ops._p(sm), ops._p(gp),
                                      None, None, ctx.stream()))
    torch.cuda.synchronize()
    assert _intact(gp, 8 * n * 256), "sentinel after g_pre overwritten"
    g_pre = gp[:8 * n * 256].view(8, n, 256)
    W16, _ = tx.weights(net, DEV)
    W16['_out32'] = net.nerf.output_linear.weight.detach().double()
    for c in vc.backward_checks(W16, scale, g, sx, g_pre):
        assert c.n_bad == 0, c.message()
    P = dict(net.nerf.named_parameters())
    t_pre = chain_torch_viewless(net, P, (sx, None, None, sm), g)[0]
    for l in range(7, 0, -1):
        k, t = g_pre[l].float(), t_pre[l].float()
        tol = 2e-2 * t.abs().amax(1, keepdim=True) + 1e-3 * t.abs()
        bad = (k - t).abs() > tol
        assert not bad.any(), ("g_pre plane", l, int(bad.sum()), float((k - t).abs().max()))


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("which", [0, 2])
def test_backward_against_torch_chain_and_fp32_autograd(nets, which, monkeypatch):
    net = copy.deepcopy(nets[which])
    pts, views = _inputs(3000, 11 + which)
    pts = pts.to(DEV)
    g = torch.randn(3000, 4, device=DEV)

    def product(torch_chain):
        if torch_chain:
            monkeypatch.setattr(autograd, "_chain_kernel", chain_torch_viewless)
            monkeypatch.setattr(autograd, "_dw_kernel", dw_torch_viewless)
        for p in net.parameters():
            p.grad = None
        x = pts.clone().requires_grad_(True)
        raw = autograd.joiner_forward(net, x, views.to(DEV))
        raw.backward(g)
        monkeypatch.undo()
        return {k: p.grad.clone() for k, p in net.nerf.named_parameters()}, x.grad.clone()
    got, gx = product(False)
    chain, cx = product(True)
    assert set(got) == {k for k, _ in net.nerf.named_parameters()}
    for k in got:
        assert torch.isfinite(got[k]).all(), k
        assert _rel(got[k], chain[k]) < 2e-3, ("kernel vs torch chain", k, _rel(got[k], chain[k]))
    assert _rel(gx, cx) < 2e-3
    # fp32 autograd through the oracle
    P = util.oracle_params(copy.deepcopy(net).to("cpu"))
    for k in P.sd:
        P.sd[k].requires_grad_(True)
    x = pts.cpu().clone().requires_grad_(True)
    no.net_forward(P, x, None).backward(g.cpu())
    for k in got:
        ref = P.sd["nerf." + k].grad
        assert _rel(got[k].cpu(), ref) < 8e-2, (k, _rel(got[k].cpu(), ref))
    assert _rel(gx.cpu(), x.grad) < 8e-2


def test_train_step_viewless_coarse_fine_matches_autograd():
    from neuman_b200 import train as nt
    c, f = viewless_net("posenc", 5)
    coarse, fine = c.to(DEV), f.to(DEV)
    opt = nb.default_opt(samples_per_ray=32, importance_samples_per_ray=32, perturb=1.0, raw_noise_std=1.0, margin=0.9,
                         use_viewdirs=False)
    R = 300
    torch.manual_seed(5)
    o = torch.randn(R, 3) * 0.1
    d = torch.nn.functional.normalize(torch.randn(R, 3), dim=-1)
    batch = dict(origin=o.to(DEV), direction=d.to(DEV), near=torch.full((R,), 0.5, device=DEV),
                 far=torch.full((R,), 4.0, device=DEV), color=torch.rand(R, 3, device=DEV),
                 depth=(1.5 + torch.rand(R)).to(DEV))
    t_rand = torch.rand(R, 32)
    noise = (torch.randn(R, 32), torch.randn(R, 64))
    kw = dict(check_bad_weights=False, penalize_empty_space=0.1, t_rand=t_rand.to(DEV), noise=tuple(x.to(DEV) for x in noise))
    losses = nt.vanilla_loss_func(coarse, fine, batch, opt, **kw)
    sum(losses).backward()
    with torch.no_grad():
        _, _, z = nb.ray_to_samples(batch, 32, perturb=1.0, t_rand=t_rand.to(DEV))
        raw_c = coarse(nb.ray_to_samples(batch, 32, perturb=1.0, t_rand=t_rand.to(DEV))[0])
        w = nb.raw2outputs(raw_c, z, batch['direction'], raw_noise_std=1.0, white_bkg=True, noise=noise[0].to(DEV))[3]
        _, _, Fz = nb.ray_to_importance_samples(batch, z, w, 32)
    z, Fz = z.cpu(), Fz.cpu()
    onets = [util.oracle_params(copy.deepcopy(coarse).cpu()), util.oracle_params(copy.deepcopy(fine).cpu())]
    for net in onets:
        for k in net.sd:
            net.sd[k].requires_grad_(True)
    import torch.nn.functional as F

    def side(net, zz, nz):
        pts = o[:, None, :] + d[:, None, :] * zz[..., None]
        raw = no.net_forward(net, pts, None)
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


# ---- 4. frame drivers against the reference goldens -------------------------------------------
def _cap(K, c2w, H, W):
    return nb.SimpleCapture(np.asarray(K), np.asarray(c2w).astype(np.float64), H, W, 0.0, 3.14)


def test_render_vanilla_against_reference(gold):
    f = util.golden("frames.npz")
    H, W, S, N = vc.VAN["H"], vc.VAN["W"], vc.VAN["S"], vc.VAN["N"]
    c, fn = (j.to(DEV) for j in vc.viewless_nets(nb.build_nerf, nb.default_opt, "posenc"))
    cap = _cap(f["van_K"], f["van_c2w"], H, W)
    rgb, dep = render.render_vanilla_range(c, cap, fn, S, N, pix0=0, n=H * W, host_out=False)
    b_rgb, b_dep = render.render_vanilla_range(c, cap, fn, S, N, pix0=0, n=H * W, host_out=False, chunk=777)
    assert torch.equal(rgb, b_rgb) and torch.equal(dep, b_dep)                       # chunk-invariant
    pix = torch.arange(H * W - 1, -1, -3, device=DEV, dtype=torch.int32)
    p_rgb, p_dep = render.render_vanilla_range(c, cap, fn, S, N, pixels=pix, host_out=False)
    assert torch.equal(p_rgb, rgb[pix.long()]) and torch.equal(p_dep, dep[pix.long()])   # pixel list = range
    e_rgb = np.abs(rgb.cpu().numpy() - gold["van_rgb"].reshape(-1, 3)).max()
    e_dep = np.abs(dep.cpu().numpy() - gold["van_depth"].reshape(-1))
    gate = max(1e-4, 1.5 * float(gold["van_floor16_depth"].max())) if util.tc_mode() else 1e-4
    assert e_rgb < TOL and (e_dep <= gate).all(), (e_rgb, float(e_dep.max()))


def _humans():
    return {k: vc.human_model(nb.HumanNeRF, nb.default_opt, k).to(DEV) for k in vc.HUMANS}


def _invariant(call, H, W):
    """A human / hybrid driver: chunk=777 and a pixel list give the range render's values."""
    a = call(pix0=0, n=H * W, host_out=False)
    b = call(pix0=0, n=H * W, host_out=False, chunk=777)
    pix = torch.arange(H * W - 1, -1, -3, device=DEV, dtype=torch.int32)
    p = call(pixels=pix, host_out=False)
    for x, y, z in zip(a, b, p):
        assert torch.equal(x, y), "chunk"
        assert torch.equal(z, x[pix.long()]), "pixel list"
    return a


def _close(a, gold, key, what, H, W, tc_floor=True):
    """rgb <= 1e-4, depth <= max(1e-4, 1.5 floor16), floor16 = the render's largest per-ray floor (the gates of
    test_gpu_render.py); grazing rays (hit / miss decided by an ill-conditioned sqrt) may flip: fewer than 1 % outliers."""
    tol = 1e-4
    if tc_floor and util.tc_mode() and (what != "rgb" or key.startswith(("hyb", "multi"))):
        tol = max(1e-4, 1.5 * float(gold[f"{key}_floor16_{what}"].max()))
    frac = vc.outliers(np.asarray(a).reshape(H * W, -1), gold[f"{key}_{what}"].reshape(H * W, -1), tol)
    assert frac < 0.01, (key, what, frac)


def test_human_renderers_against_reference(gold):
    f = util.golden("frames.npz")
    H, W, S, N = vc.HUM["H"], vc.HUM["W"], vc.HUM["S"], vc.HUM["N"]
    cap = _cap(f["h_K"], f["h_c2w"], H, W)
    b1 = synth_smpl.random_body(seed=1, center=(0.1, 0.0, 0.3))
    b2 = synth_smpl.random_body(seed=4, center=(-0.15, 0.0, 0.5))
    geo = b1["geo_threshold"]
    models = _humans()
    for k, m in models.items():
        sums = [vc.checksum(j) for j in (m.coarse_bkg_net, m.fine_bkg_net, m.coarse_human_net)]
        assert np.allclose(np.array(sums), gold[f"human{k}_sums"], rtol=1e-9, atol=0), k      # summed on the device
    A = models["A"]
    for can in (1, 0):
        r, d, a = _invariant(lambda **kw: render.render_smpl_nerf_range(A, cap, b1["verts"], b1["faces"], b1["Ts"], S,
                                                                         render_can=bool(can), geo_threshold=geo, **kw), H, W)
        _close(r.cpu(), gold, f"smpl{can}", "rgb", H, W)
        _close(d.cpu(), gold, f"smpl{can}", "depth", H, W)
        _close(a.cpu(), gold, f"smpl{can}", "acc", H, W)
    for k, m in models.items():
        r, d, _ = _invariant(lambda **kw: render.render_hybrid_nerf_range(m, cap, b1["verts"], b1["faces"], b1["Ts"], S, N,
                                                                           geo_threshold=geo, **kw), H, W)
        _close(r.cpu(), gold, f"hyb{k}", "rgb", H, W)
        _close(d.cpu(), gold, f"hyb{k}", "depth", H, W)
    r, d = nb.render_hybrid_nerf_multi_persons(A, cap, [A, models["B"]], [b1["verts"], b2["verts"]], [b1["faces"], b2["faces"]],
                                               [b1["Ts"], b2["Ts"]], samples_per_ray=S, importance_samples_per_ray=N,
                                               geo_threshold=geo, return_depth=True)
    _close(r, gold, "multi", "rgb", H, W)
    _close(d, gold, "multi", "depth", H, W)
    # the multi-person driver: chunk and pixel-list invariance with one actor of each kind
    hm, vs, fs, ts = [A, models["B"]], [b1["verts"], b2["verts"]], [b1["faces"], b2["faces"]], [b1["Ts"], b2["Ts"]]
    r0, d0, _ = _invariant(lambda pix0=0, n=None, host_out=False, chunk=render.CHUNK, pixels=None:
                           render._hybrid(A, hm, cap, vs, fs, ts, S, N, True, geo, True, pix0, n, host_out, chunk, pixels=pixels),
                           H, W)
    assert np.array_equal(r0.cpu().numpy().reshape(H, W, 3), r) and np.array_equal(d0.cpu().numpy().reshape(H, W), d)


# ---- 5. slot kind switching -------------------------------------------------------------------
def test_slot_switches_kind():
    """One slot packed view -> view-independent -> view: forward and backward equal those of fresh slots."""
    ctx = ops._ctx_for(torch.zeros(1, device=DEV))
    view, _ = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False), 8)
    vl, _ = viewless_net("rotate", 9)
    view, vl = view.to(DEV), vl.to(DEV)
    pts, views = _inputs(2000, 3)
    pts, views = pts.to(DEV), views.to(DEV)
    g = torch.randn(2000, 4, device=DEV)

    def run(j):
        raw = ops.joiner_forward(j, pts, views, mode=MODES["tc"])
        for p in j.parameters():
            p.grad = None
        autograd.joiner_forward(j, pts, views).backward(g)
        return raw, {k: p.grad.clone() for k, p in j.nerf.named_parameters()}
    fresh = {id(j): run(j) for j in (view, vl)}
    saved = (dict(ctx.slots), list(ctx.slot_keys), list(ctx.slot_used))
    try:
        for j in (view, vl, view):
            ops.invalidate_net(j)
            ctx.slots = {}
            ctx.slot_keys = [None] + [("held",)] * (len(ctx.slot_keys) - 1)    # the only free slot: 0
            assert ops.net_slot(j, ctx) == 0
            raw, grads = run(j)
            assert torch.equal(raw, fresh[id(j)][0])
            for k in grads:                     # the weight-gradient kernel reduces with atomics: summation order varies
                assert _rel(grads[k], fresh[id(j)][1][k]) < 1e-5, k
    finally:
        slots, keys, used = saved
        ctx.slots = {k: v for k, v in slots.items() if v != 0}               # slot 0 now holds `view`: forget it
        ctx.slot_keys = [None if i == 0 else k for i, k in enumerate(keys)]
        ctx.slot_used = used
        for j in (view, vl):
            ops.invalidate_net(j)


# ---- 6. range guard ---------------------------------------------------------------------------
def test_range_guard():
    ctx = ops._ctx_for(torch.zeros(1, device=DEV))
    ctx.range_check(clear=True)
    j, _ = viewless_net("posenc", 12, boost=False)
    with torch.no_grad():
        for lin in j.nerf.pts_linears:
            lin.weight.mul_(40.0)
    j = j.to(DEV)
    pts, _ = _inputs(20000, 4)
    ops.joiner_forward(j, pts.to(DEV) * 3, None, mode=MODES["tc"])
    with pytest.raises(_lib.NmError, match="-5"):
        ctx.range_check(clear=True)


# ---- 7. drop-in -------------------------------------------------------------------------------
def test_dropin_runs_viewless_calls_on_the_library():
    """Under install() the stand-in reference's render_vanilla (view-independent coarse + fine) and render_hybrid_nerf
    (view background + specular_can=False human) run on the library: the reference functions are wrapped in spies before
    install() stashes them, and the spies are never called; the results match the reference goldens."""
    from tests.standin_reference import standin
    f = util.golden("frames.npz")
    gold = util.golden("viewless.npz")
    with standin() as r:
        calls = []
        for name in ("render_vanilla", "render_hybrid_nerf"):
            orig = getattr(r.render_utils, name)

            def spy(*a, _orig=orig, _name=name, **k):
                calls.append(_name)
                return _orig(*a, **k)
            setattr(r.render_utils, name, spy)
        nb.install()
        try:
            c, fn = vc.viewless_nets(r.vanilla.build_nerf, nb.default_opt, "posenc")
            c, fn = c.to(DEV), fn.to(DEV)
            assert type(c).__module__ == "models.vanilla" and nb.dropin.supported_joiner(c)
            H, W, S, N = vc.VAN["H"], vc.VAN["W"], vc.VAN["S"], vc.VAN["N"]
            l0 = ops.Context.get(0).launch_count()
            with torch.no_grad():
                rgb = r.render_utils.render_vanilla(c, _cap(f["van_K"], f["van_c2w"], H, W), fine_net=fn, rays_per_batch=100,
                                                    samples_per_ray=S, importance_samples_per_ray=N)
                raw = c(torch.zeros(5, 3, device=DEV))                 # Joiner.forward without views
            assert ops.Context.get(0).launch_count() > l0 and raw.shape == (5, 4) and raw.is_cuda
            assert np.abs(rgb - gold["van_rgb"]).max() < TOL
            human = vc.human_model(nb.HumanNeRF, nb.default_opt, "A").to(DEV)
            assert not human.coarse_human_net.nerf.use_viewdirs
            b1 = synth_smpl.random_body(seed=1, center=(0.1, 0.0, 0.3))
            H, W, S, N = vc.HUM["H"], vc.HUM["W"], vc.HUM["S"], vc.HUM["N"]
            with torch.no_grad():
                rh, dh = r.render_utils.render_hybrid_nerf(human, _cap(f["h_K"], f["h_c2w"], H, W), b1["verts"], b1["faces"],
                                                           b1["Ts"], rays_per_batch=64, samples_per_ray=S,
                                                           importance_samples_per_ray=N, geo_threshold=b1["geo_threshold"],
                                                           return_depth=True)
            _close(rh, gold, "hybA", "rgb", H, W)
            _close(dh, gold, "hybA", "depth", H, W)
            assert calls == [], calls                                  # the reference functions were never reached
        finally:
            nb.dropin.uninstall()
