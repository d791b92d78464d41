"""Element-by-element checks of the tensor-core MLP kernels against exact fp16-operand arithmetic (tests/tc_exact.py):
the training forward's activation stash, sign words and raw outputs, the backward chain's gradient planes, the fp16
encodings and the encoding adjoint.  Every element must lie in its proven window; nothing is compared at a tuned
tolerance.  Also: sentinel regions after every output buffer stay untouched at ragged sizes, and a backward chain that
overflows fp16 reaches the gradients as non-finite values, which the training step's device guard then skips."""
import copy

import pytest
import torch

import neuman_b200 as nb
from neuman_b200 import _lib, ops
from neuman_b200.autograd import _encodings, _pow2_scale
from neuman_b200.ops import _p
from tests import tc_exact as tx
from tests import util
from tests.test_tc_exact import carrier_joiner

pytestmark = pytest.mark.gpu
DEV = "cuda"
PAD_ROWS = 128          # sentinel rows after every output plane: one whole tile


def _T():
    """rows per wave of the persistent kernels: 128-sample tiles x one CTA per SM"""
    return 128 * torch.cuda.get_device_properties(0).multi_processor_count


SIZES = [1, 63, 64, 65, 127, 128, 129, 4173, "T", "T+1", "3T-5"]


def _n(size):
    return {"T": _T(), "T+1": _T() + 1, "3T-5": 3 * _T() - 5}.get(size, size)


@pytest.fixture(scope="module")
def nets():
    coarse, _, human = util.product_nets(DEV)
    x3 = copy.deepcopy(coarse)
    with torch.no_grad():
        for name, p in x3.nerf.named_parameters():
            if name.endswith("weight"):
                p.mul_(3.0)
    return {"coarse": coarse, "human": human, "carrier": carrier_joiner().to(DEV), "coarse_x3": x3}


class Guarded:
    """An output buffer followed by PAD_ROWS rows of a sentinel bit pattern; .t is the [shape] view handed to the kernel."""

    def __init__(self, shape, dtype, bits):
        rows, row = shape[-2], shape[-1]
        used = 1
        for s in shape:
            used *= s
        self.used = used
        self.buf = torch.empty(used + PAD_ROWS * row, dtype=dtype, device=DEV)
        ib = {torch.float16: torch.int16, torch.float32: torch.int32, torch.int32: torch.int32}[dtype]
        self.ib, self.bits = ib, bits
        self.buf.view(ib).fill_(bits)
        self.t = self.buf[:used].view(*shape)

    def intact(self):
        return bool((self.buf[self.used:].view(self.ib) == self.bits).all())


def forward_train(j, pts, views):
    """nm_mlp_forward_train through ctypes into guarded buffers -> dict of Guarded (raw, sx, sf, sv, sm)."""
    ctx = ops._ctx_for(pts)
    slot = ops.net_slot(j, ctx)
    n = pts.shape[0]
    o = dict(raw=Guarded((n, 4), torch.float32, -1), sx=Guarded((8, n, 256), torch.float16, -1),
             sf=Guarded((n, 256), torch.float16, -1), sv=Guarded((n, 128), torch.float16, -1),
             sm=Guarded((9, n, 8), torch.int32, -1))
    ctx.check(ctx.lib.nm_mlp_forward_train(ctx.h, slot, _p(pts), _p(views), n, 0, _p(o['raw'].t), _p(o['sx'].t), _p(o['sf'].t),
                                           _p(o['sv'].t), _p(o['sm'].t), ctx.stream()))
    return o


def backward(j, d_raw, scale, sv, sm):
    ctx = ops._ctx_for(d_raw)
    slot = ops.net_slot(j, ctx)
    n = d_raw.shape[0]
    o = dict(g_pre=Guarded((8, n, 256), torch.float16, -1), g_f=Guarded((n, 256), torch.float16, -1),
             g_v=Guarded((n, 128), torch.float16, -1))
    ctx.check(ctx.lib.nm_mlp_backward(ctx.h, slot, _p(d_raw), _p(scale), n, _p(sv), _p(sm), _p(o['g_pre'].t), _p(o['g_f'].t),
                                      _p(o['g_v'].t), ctx.stream()))
    return o


def _inputs(n, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    pts = torch.randn(n, 3, device=DEV, generator=g) * 1.5
    views = torch.nn.functional.normalize(torch.randn(n, 3, device=DEV, generator=g), dim=-1)
    return pts, views, torch.randn(n, 4, device=DEV, generator=g)


def _report(tag, checks):
    occ = " ".join(f"{c.name}={c.occupancy:.4f}" for c in checks)
    print(f"\n[tc_exact] {tag} window occupancy: {occ}")
    for c in checks:
        if c.name in ("rgb", "alpha"):
            used = float(((c.v - c.e).abs() / c.B.clamp_min(1e-300)).max())
            print(f"[tc_exact] {tag} {c.name}: max |v - e| / B = {used:.4f}")


@pytest.mark.parametrize("net", ["coarse", "human", "carrier", "coarse_x3"])
@pytest.mark.parametrize("size", SIZES)
def test_training_forward_and_backward_in_exact_windows(nets, net, size):
    """Every element of sx, sf, sv, raw (forward) and g_v, g_f, g_pre (backward, on the kernel's own stash and
    gradient planes) lies in its window; the sign words equal the layout built from (sx > 0) and (sv > 0); the
    inference kernel's raw is bit-identical to the training raw; the sentinels after every buffer are untouched."""
    j = nets[net]
    n = _n(size)
    pts, views, d_raw = _inputs(n, n)
    ctx = _lib.Context.get(0)
    ctx.range_check()                                           # clear
    o = forward_train(j, pts, views)
    raw, sx, sf, sv, sm = (o[k].t for k in ("raw", "sx", "sf", "sv", "sm"))
    pe, dpe = _encodings(j, pts, views)
    W16, W32 = tx.weights(j, DEV)
    checks = list(tx.forward_checks(W16, W32, pe, dpe, sx, sf, sv, raw))
    for c in checks:
        assert c.ok.all(), (net, n, c.message())
    votes, rows = tx.alpha_input_votes(W16, W32, pe, sx, raw)
    assert votes < 0.05 or rows < 20, (net, n, "alpha head follows the rounded layer 7", votes, rows)
    # sign words: planes 0..7 from sx, plane 8 (words 0..3) from sv
    m = sm.to(torch.int64) & 0xFFFFFFFF
    for l in range(8):
        assert torch.equal(m[l], tx.sign_words(sx[l])), (net, n, "sign words of layer", l)
    assert torch.equal(m[8, :, :4], tx.sign_words(sv)), (net, n, "sign words of the views layer")
    # the inference kernel computes the same raw, bit for bit
    inf_raw = ops.joiner_forward(j, pts, views, mode=_lib.NM_MLP_TC_F16)
    assert torch.equal(inf_raw, raw), (net, n)
    ctx.range_check()                                           # raises if an activation reached the fp16 limit
    for k, g in o.items():
        assert g.intact(), (net, n, k, "sentinel after the buffer overwritten")
    # backward chain
    scale = _pow2_scale(d_raw, 256.0)
    b = backward(j, d_raw, scale, sv, sm)
    bchecks = list(tx.backward_checks(W16, W32, float(scale), d_raw, sx, sv, b['g_pre'].t, b['g_f'].t, b['g_v'].t))
    for c in bchecks:
        assert c.ok.all(), (net, n, c.message())
    for k, g in b.items():
        assert g.intact(), (net, n, k, "sentinel after the buffer overwritten")
    if n >= 4173:
        _report(f"{net} n={n}", checks + bchecks)


def _special_points(emb, n_rand):
    """|x| up to 100, x = 0, and points whose encoding argument lands next to a multiple of pi (sin ~ 0)."""
    g = torch.Generator().manual_seed(5)
    pts = [torch.randn(n_rand, 3, generator=g) * 1.5, (torch.rand(n_rand, 3, generator=g) * 2 - 1) * 100.0,
           torch.zeros(4, 3)]
    tab = tx.encoder_table(emb)
    m = torch.arange(1, 9, dtype=torch.float64)
    if emb.mapping == 'rotate':
        for b in tab:                                           # x . b = m pi
            pts.append((m[:, None] * torch.pi * b[None] / float(b @ b)).float())
    else:
        for f in tab:
            for d in range(3):
                x = torch.zeros(len(m), 3, dtype=torch.float64)
                x[:, d] = m * torch.pi / f
                pts.append(x.float())
    return torch.cat(pts).float()


@pytest.mark.parametrize("kind", ["posenc", "rotate"])
def test_encodings_equal_rounded_float64_embedder(kind):
    """nm_encode_f16 (the encoder of k_mlp_tc, exact cycle reduction + MUFU sin/cos) equals r16 of the float64
    Embedder within the MUFU error and the reduction error (tc_exact.encoder_delta); the raw input channels are exactly
    r16(x), the constant channel exactly 1, the padding exactly 0.  Position and direction encoders, per-sample and
    grouped inputs."""
    j, _ = util.scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False, posenc=kind), 3)
    j = j.to(DEV)
    ctx = _lib.Context.get(0)
    slot = ops.net_slot(j, ctx)
    for which, emb, width in ((0, j.pos_pe, 64), (1, j.dir_pe, 32)):
        x = _special_points(emb, 3000).to(DEV)
        for group in (0, 3):
            n = x.shape[0] * (group or 1)
            out = torch.empty(n, width, device=DEV, dtype=torch.float16)
            ctx.check(ctx.lib.nm_encode_f16(ctx.h, slot, which, _p(x), group, n, _p(out), ctx.stream()))
            xr = x.repeat_interleave(group, 0) if group else x
            c = tx.encoding_check(f"{kind} which={which} group={group}", out, xr, emb, width)
            assert c.ok.all(), c.message()
            print(f"\n[tc_exact] encoder {kind} which={which}: window occupancy {c.occupancy:.4f}")


@pytest.mark.parametrize("kind", ["posenc", "rotate"])
@pytest.mark.parametrize("group,inv", [(0, None), (4, 2.0 ** -7)])
def test_pe_backward_against_float64_jacobian(kind, group, inv):
    """nm_pe_backward (fp32, accurate sincosf) against the float64 Jacobian of Embedder.forward applied to d_enc, within
    the bound of an fp32 evaluation (tc_exact.pe_backward_ref: relative to sum_c |d_enc_c d enc_c / dx| plus the fp32
    argument's rounding).  Both encoders, grouped inputs, the inv_scale argument."""
    j, _ = util.scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False, posenc=kind), 4)
    j = j.to(DEV)
    ctx = _lib.Context.get(0)
    slot = ops.net_slot(j, ctx)
    gen = torch.Generator(device=DEV).manual_seed(11)
    for which, emb, ld in ((0, j.pos_pe, 64), (1, j.dir_pe, 32)):
        rows = 2000
        x = torch.cat([torch.randn(rows, 3, device=DEV, generator=gen) * 1.5,
                       (torch.rand(rows, 3, device=DEV, generator=gen) * 2 - 1) * 100.0])
        n = x.shape[0] * (group or 1)
        d_enc = torch.randn(n, ld, device=DEV, generator=gen) * 3.0
        inv_t = torch.full((1,), inv, device=DEV) if inv is not None else None
        d_x = torch.empty(n, 3, device=DEV)
        ctx.check(ctx.lib.nm_pe_backward(ctx.h, slot, which, _p(x), group, _p(d_enc), ld, _p(inv_t), n, _p(d_x), ctx.stream()))
        xr = x.repeat_interleave(group, 0) if group else x
        ref, B = tx.pe_backward_ref(xr, emb, d_enc, inv if inv is not None else 1.0)
        bad = (d_x.double() - ref).abs() > B
        assert not bad.any(), (kind, which, int(bad.sum()), float(((d_x.double() - ref).abs() / B).max()))


def _f64_chain(j, pts, views, d_raw):
    """max |activation| of the float64 forward and max |S * gradient| of the float64 backward chain."""
    P = {k: v.detach().double() for k, v in j.nerf.state_dict().items()}
    pe, ve = tx.embed64(pts, j.pos_pe), tx.embed64(views, j.dir_pe)
    h, acts = pe, []
    for l in range(8):
        h = torch.relu(h @ P[f'pts_linears.{l}.weight'].T + P[f'pts_linears.{l}.bias'])
        acts.append(h)
        if l == 4:
            h = torch.cat([pe, h], 1)
    f = h @ P['feature_linear.weight'].T + P['feature_linear.bias']
    v = torch.relu(torch.cat([f, ve], 1) @ P['views_linears.0.weight'].T + P['views_linears.0.bias'])
    fmax = max(float(a.abs().max()) for a in acts + [f, v])
    gs = float(_pow2_scale(d_raw, 256.0)) * d_raw.double()
    g = (gs[:, :3] @ P['rgb_linear.weight']) * (v > 0)
    gmax = float(g.abs().max())
    g = g @ P['views_linears.0.weight'][:, :256]
    dX = g @ P['feature_linear.weight'] + gs[:, 3:4] * P['alpha_linear.weight']
    for l in range(7, -1, -1):
        g = dX * (acts[l] > 0)
        gmax = max(gmax, float(g.abs().max()))
        if l > 0:
            w = P[f'pts_linears.{l}.weight']
            dX = g @ (w[:, 63:] if l == 5 else w)
    return fmax, gmax


def test_backward_overflow_reaches_the_gradients_and_the_device_guard_skips_the_step():
    """Weights scaled so that the forward stays in the fp16 range (range flag clear) while the float64 backward chain
    exceeds 65504 (factor found here from the float64 chain).  The chain's packs do not saturate: every element whose
    exact value is beyond the fp16 range is +-inf (the windows demand it), the parameter gradients are non-finite, and
    train_batch(nan_guard='device') leaves the parameters and Adam's moments exactly as they were."""
    from neuman_b200 import train as nt
    coarse, _, _ = util.product_nets(DEV)
    n = 4096
    pts, views, d_raw = _inputs(n, 21)
    factor = None
    for k in (4.0, 4.5, 5.0, 5.5, 6.0):
        j = copy.deepcopy(coarse)
        with torch.no_grad():
            for name, p in j.nerf.named_parameters():
                if name.endswith("weight"):
                    p.mul_(k)
        fmax, gmax = _f64_chain(j, pts, views, d_raw)
        if fmax < 65504 / 2 and gmax > 2 * 65504:
            factor = k
            break
    assert factor is not None, "no weight scale keeps the forward in range and overflows the chain"
    print(f"\n[tc_exact] overflow factor {factor}: forward max {fmax:.1f}, float64 chain max {gmax:.1f}")
    ctx = _lib.Context.get(0)
    ctx.range_check()
    o = forward_train(j, pts, views)
    sx, sv, sm = o['sx'].t, o['sv'].t, o['sm'].t
    ctx.range_check()                                           # the forward stayed in range
    scale = _pow2_scale(d_raw, 256.0)
    b = backward(j, d_raw, scale, sv, sm)
    W16, W32 = tx.weights(j, DEV)
    required_inf = 0
    for c in tx.backward_checks(W16, W32, float(scale), d_raw, sx, sv, b['g_pre'].t, b['g_f'].t, b['g_v'].t):
        fin = torch.isfinite(c.e)                               # rows whose input plane already overflowed have no reference
        assert c.ok[fin].all(), c.message()
        required_inf += int((torch.isinf(c.lo) & fin).sum())         # there v must be inf: 65504 would fail the window
    assert required_inf > 0
    # through autograd: the parameter gradients are not finite
    j.zero_grad()
    (j(pts, views) * d_raw).sum().backward()
    assert not all(bool(torch.isfinite(p.grad).all()) for p in j.nerf.parameters())
    # the training step: a normal step on the unscaled net fills Adam's state, then the weights are scaled in place
    net = copy.deepcopy(coarse)
    opt = nb.default_opt(samples_per_ray=32, importance_samples_per_ray=0, perturb=0.0, raw_noise_std=0.0)
    R = 128
    gen = torch.Generator(device=DEV).manual_seed(3)
    batch = dict(origin=torch.randn(R, 3, device=DEV, generator=gen) * 0.1,
                 direction=torch.nn.functional.normalize(torch.randn(R, 3, device=DEV, generator=gen), dim=-1),
                 near=torch.full((R,), 0.5, device=DEV), far=torch.full((R,), 3.0, device=DEV),
                 color=torch.rand(R, 3, device=DEV, generator=gen))
    optim = torch.optim.Adam(net.parameters(), lr=5e-4)
    loss = nt.train_batch(net, None, optim, batch, opt, check_bad_weights=False)
    assert torch.isfinite(loss)
    # the loss concentrates dL/d raw on few samples, so this batch may need a larger scale than random d_raw: the smallest
    # one whose chain overflows (precondition of what follows)
    for f in (factor, 6.0, 7.0, 8.0, 10.0):
        probe = copy.deepcopy(net)
        with torch.no_grad():
            for name, p in probe.nerf.named_parameters():
                if name.endswith("weight"):
                    p.mul_(f)
        probe.zero_grad()
        sum(nt.vanilla_loss_func(probe, None, batch, opt, check_bad_weights=False)).backward()
        if not all(bool(torch.isfinite(p.grad).all()) for p in probe.nerf.parameters()):
            break
    else:
        pytest.fail("no weight scale overflows the chain on the training batch")
    try:
        ctx.range_check()                   # cleared: at this scale the forward may saturate; the in-range case is above
    except _lib.NmError:
        pass
    with torch.no_grad():
        for name, p in net.nerf.named_parameters():
            if name.endswith("weight"):
                p.mul_(f)
    before = {k: p.detach().clone() for k, p in net.named_parameters()}
    state = {k: {s: t.clone() for s, t in optim.state[p].items()} for k, p in net.named_parameters()}
    loss = nt.train_batch(net, None, optim, batch, opt, check_bad_weights=False, nan_guard='device')
    for k, p in net.named_parameters():
        assert torch.equal(p.detach(), before[k]), (k, "parameter moved on a skipped step")
        for s in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(optim.state[p][s], state[k][s]), (k, s)
