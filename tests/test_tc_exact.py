"""The exact-window rule of tests/tc_exact.py, checked on the CPU: an fp32 evaluation of the tensor-core kernels'
arithmetic (fp16 operands, fp32 accumulation in two different orders, fp16 rounding to nearest) is accepted everywhere,
and each planted defect of the kind a kernel rewrite can introduce is rejected on a clear majority of the elements it
changes.  This is what gives the GPU gates of tests/test_gpu_tc_exact.py their meaning."""
import pytest
import torch

from tests import tc_exact as tx
from tests import util

N = 1024
DEFECTS = ("swizzle_slip", "bias_dropped", "round_toward_zero", "alpha_from_rounded", "rgb_bias_f16")


def carrier_joiner():
    """The offset net's carrier Joiner (models.offset_joiner_weights): any-sign output through +-W, a unit views layer."""
    import neuman_b200 as nb
    from neuman_b200 import models
    torch.manual_seed(9)
    net = nb.build_offset_net(nb.default_opt(use_cuda=False, num_offset_nets=1))
    j = models.offset_shadow_joiner(net)
    W = models.offset_joiner_weights(net, 0.4)
    with torch.no_grad():
        for k, p in j.nerf.named_parameters():
            p.copy_(W[k])
    return j


def nets():
    coarse, _, human = util.product_nets("cpu")
    return {"coarse": coarse, "human": human, "carrier": carrier_joiner()}


def _mm32(a, W, order):
    """fp32 a @ W^T: torch's own order, or K reversed in blocks of 16 (the wgmma K step) summed last block first."""
    a, W = a.float(), W.float()
    if order == "plain":
        return a @ W.T
    acc = torch.zeros(a.shape[0], W.shape[0])
    K = a.shape[1]
    for k0 in reversed(range(0, K, 16)):
        acc = acc + a[:, k0:k0 + 16].flip(1) @ W[:, k0:k0 + 16].flip(1).T
    return acc


def _rz16(x):
    """fp32 -> fp16 rounding toward zero"""
    h = x.half()
    bits = h.view(torch.int16).clone()
    away = h.float().abs() > x.abs()
    bits[away] -= 1
    return bits.view(torch.float16)


def encodings(j, pts, views):
    """fp16 encodings laid out like nm_encode_f16: [n,64] with channel 63 = 1, [n,32] with channel 27 = 1."""
    pe, dpe = torch.zeros(pts.shape[0], 64), torch.zeros(pts.shape[0], 32)
    pe[:, :63] = tx.r16(tx.embed64(pts, j.pos_pe)).float()
    dpe[:, :27] = tx.r16(tx.embed64(views, j.dir_pe)).float()
    pe[:, 63] = 1.0
    dpe[:, 27] = 1.0
    return pe.half(), dpe.half()


def emulate_forward(j, pe, dpe, order="plain", defect=None):
    """The training forward's arithmetic in fp32 on the CPU -> sx, sf, sv, raw (fp16 planes, fp32 raw)."""
    sd = {k: v.detach() for k, v in j.nerf.state_dict().items()}
    h16 = {k: v.half() for k, v in sd.items()}
    n = pe.shape[0]
    sx = torch.empty(8, n, 256, dtype=torch.float16)
    acc7 = None
    for l in range(8):
        w, b = h16[f'pts_linears.{l}.weight'].clone(), h16[f'pts_linears.{l}.bias']
        a = pe[:, :63] if l == 0 else (torch.cat([pe[:, :63], sx[4]], 1) if l == 5 else sx[l - 1])
        if defect == "swizzle_slip" and l == 3:
            w[:, [40, 41]] = w[:, [41, 40]]
        acc = _mm32(a, w, order)
        if not (defect == "bias_dropped" and l == 2):
            acc = acc + b.float()
        out = torch.relu(acc)
        sx[l] = _rz16(out) if (defect == "round_toward_zero" and l == 6) else out.half()
        if l == 7:
            acc7 = acc
    sf = (_mm32(sx[7], h16['feature_linear.weight'], order) + h16['feature_linear.bias'].float()).half()
    a = torch.cat([sf, dpe[:, :27]], 1)
    sv = torch.relu(_mm32(a, h16['views_linears.0.weight'], order) + h16['views_linears.0.bias'].float()).half()
    rgb_b = sd['rgb_linear.bias'].half().float() if defect == "rgb_bias_f16" else sd['rgb_linear.bias']
    rgb = _mm32(sv, h16['rgb_linear.weight'], order) + rgb_b
    r7 = sx[7].float() if defect == "alpha_from_rounded" else torch.relu(acc7)
    alpha = r7 @ sd['alpha_linear.weight'][0] + sd['alpha_linear.bias']
    return sx, sf, sv, torch.cat([rgb, alpha[:, None]], 1)


def emulate_backward(j, sx, sv, d_raw, scale, order="plain"):
    """The backward chain's arithmetic in fp32 on the CPU -> g_pre, g_f, g_v (fp16)."""
    sd = {k: v.detach() for k, v in j.nerf.state_dict().items()}
    gs = d_raw * scale
    g_v = ((gs[:, :3] @ sd['rgb_linear.weight']) * (sv > 0)).half()
    g_f = _mm32(g_v, sd['views_linears.0.weight'][:, :256].T.half(), order).half()
    dX = _mm32(g_f, sd['feature_linear.weight'].T.half(), order) + gs[:, 3:4] * sd['alpha_linear.weight']
    g_pre = torch.empty_like(sx)
    for l in range(7, -1, -1):
        g_pre[l] = (dX * (sx[l] > 0)).half()
        if l > 0:
            w = sd[f'pts_linears.{l}.weight']
            w = w[:, 63:] if l == 5 else w
            dX = _mm32(g_pre[l], w.T.half(), order)
    return g_pre, g_f, g_v


def _inputs(seed):
    torch.manual_seed(seed)
    pts = torch.randn(N, 3) * 1.5
    views = torch.nn.functional.normalize(torch.randn(N, 3), dim=-1)
    return pts, views


def _forward_checks(j, pe, dpe, outs):
    W16, W32 = tx.weights(j, "cpu")
    return {c.name: c for c in tx.forward_checks(W16, W32, pe, dpe, *outs)}


@pytest.mark.parametrize("net", ["coarse", "human", "carrier"])
@pytest.mark.parametrize("order", ["plain", "reversed_blocked"])
def test_rule_accepts_fp32_evaluations(net, order):
    """Every element of every forward and backward output of an fp32 evaluation lies in its window."""
    j = nets()[net]
    pts, views = _inputs(1)
    pe, dpe = encodings(j, pts, views)
    outs = emulate_forward(j, pe, dpe, order)
    for c in _forward_checks(j, pe, dpe, outs).values():
        assert c.ok.all(), c.message()
    votes, rows = tx.alpha_input_votes(*tx.weights(j, "cpu"), pe, outs[0], outs[3])
    assert votes < 0.05 or rows < 10, (votes, rows)
    sx, sf, sv, raw = outs
    torch.manual_seed(2)
    d_raw = torch.randn(N, 4)
    from neuman_b200.autograd import _pow2_scale
    scale = float(_pow2_scale(d_raw, 256.0))
    W16, W32 = tx.weights(j, "cpu")
    for c in tx.backward_checks(W16, W32, scale, d_raw, sx, sv, *emulate_backward(j, sx, sv, d_raw, scale, order)):
        assert c.ok.all(), c.message()


@pytest.mark.parametrize("defect", DEFECTS)
def test_rule_rejects_planted_defects(defect):
    """Each defect is rejected on a clear majority (> 2/3) of the elements it changes, and only in its own layer (the
    checks are layer-local: later layers see the defective plane as their input).  The alpha head on the rounded layer 7
    stays inside the alpha window (which has to carry layer 7's bound through |w_alpha|): tc_exact.alpha_input_votes
    catches it instead, on nearly every row where the two models differ."""
    layer = {"swizzle_slip": "layer3", "bias_dropped": "layer2", "round_toward_zero": "layer6",
             "alpha_from_rounded": "alpha", "rgb_bias_f16": "rgb"}[defect]
    j = nets()["coarse"]
    pts, views = _inputs(3)
    pe, dpe = encodings(j, pts, views)
    good = emulate_forward(j, pe, dpe)
    bad = emulate_forward(j, pe, dpe, defect=defect)
    checks = _forward_checks(j, pe, dpe, bad)
    names = ["layer%d" % l for l in range(8)] + ["feature", "views", "rgb", "alpha"]
    planes = dict(zip(names, list(bad[0]) + [bad[1], bad[2], bad[3][:, :3], bad[3][:, 3]]))
    ref_planes = dict(zip(names, list(good[0]) + [good[1], good[2], good[3][:, :3], good[3][:, 3]]))
    for name, c in checks.items():
        if name != layer:
            continue
        if defect == "alpha_from_rounded":
            votes, rows = tx.alpha_input_votes(*tx.weights(j, "cpu"), pe, bad[0], bad[3])
            print(f"{defect}: {rows} rows separate the two head models, {votes:.3f} vote for the rounded input")
            assert rows > 100 and votes > 0.9, (votes, rows)
            continue
        # the inputs of the defective layer are the good evaluation's, so `affected` is what the defect changed
        affected = planes[name] != ref_planes[name]
        assert int(affected.sum()) > 0, (defect, "the defect changes nothing")
        rejected = float((~c.ok & affected).sum()) / float(affected.sum())
        print(f"{defect}: {name} changed {int(affected.sum())} elements, rejected {rejected:.3f}")
        assert rejected > 2 / 3, (defect, name, rejected)
    for name, c in checks.items():
        if name != layer and not (defect == "alpha_from_rounded"):
            assert c.ok.all(), (defect, c.message())
