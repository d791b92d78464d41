"""Element-by-element checks of the weight and bias gradients of the tensor-core training step against float64 windows
(tests/dw_exact.py): nm_dw_gemm launched directly on adversarial planes, and every parameter gradient of Joiner.forward
under torch autograd for every net kind, on the planes the step itself used.  Every element must lie in its proven
window; nothing is compared at a tuned tolerance.  All float64 references run on the GPU."""
import pytest
import torch

from neuman_b200 import autograd as nag
from neuman_b200 import ops
from neuman_b200.ops import _p
from tests import dw_exact as dx
from tests import tc_exact as tx
from tests.test_dw_exact import kind_inputs, kind_nets
from tests.test_gpu_tc_exact import Guarded

pytestmark = pytest.mark.gpu
DEV = "cuda"
STEP = 2048 * 128 + 77                  # one coarse training step's samples, ragged


def _sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pairs():
    return min(_sm() // 2, dx.DW_MAX_WORK)


DIRECT_SIZES = [1, 63, 64, 65, 640, "P-1", "P+1", "2P-1", "2P+1", 4173, 14213, STEP]


def _n_direct(size):
    P = 64 * _pairs()
    return {"P-1": P - 1, "P+1": P + 1, "2P-1": 2 * P - 1, "2P+1": 2 * P + 1}.get(size, size)


@pytest.mark.parametrize("trunk_only", [False, True])
@pytest.mark.parametrize("size", DIRECT_SIZES)
def test_dw_gemm_in_exact_windows(size, trunk_only):
    """nm_dw_gemm on adversarial planes: every element of dw and db lies in dw_window; rows 128..255 of item 8 are
    exactly 0; in the trunk-only launch (g_f = g_v = sf = NULL, a view-independent net) planes 7 and 8 are exactly 0; the
    sentinels after both outputs are intact.  n = 64 k pairs +- 1 straddles the work split of this GPU's CTA pairs."""
    n = _n_direct(size)
    planes = dx.dw_planes(n, 1000 + n, DEV)
    ctx = ops._ctx_for(planes['g_f'])
    out = Guarded((9, 256, 256), torch.float32, -1)
    bias = Guarded((9, 256), torch.float32, -1)
    g_f, g_v, sf = (None, None, None) if trunk_only else (planes['g_f'], planes['g_v'], planes['sf'])
    ctx.check(ctx.lib.nm_dw_gemm(ctx.h, _p(planes['g_pre']), _p(g_f), _p(g_v), _p(planes['sx']), _p(sf), n,
                                 _p(out.t), _p(bias.t), ctx.stream()))
    dw, db = out.t, bias.t
    items = dx.dw_items(planes, trunk_only)
    use = []
    for k, (G, X) in enumerate(items):
        m = G.shape[1]
        e, B = dx.dw_window(G, X)
        dx.assert_in_window(f"dw item {k} n={n}", dw[k, :m], e, B)
        eb, Bb = dx.dw_window(G, None)
        dx.assert_in_window(f"db item {k} n={n}", db[k, :m], eb[:, 0], Bb[:, 0])
        use.append(dx.used(dw[k, :m], e, B))
    assert torch.equal(dw[8, 128:], torch.zeros_like(dw[8, 128:])) and torch.equal(db[8, 128:], torch.zeros_like(db[8, 128:]))
    if trunk_only:
        assert torch.equal(dw[7:], torch.zeros_like(dw[7:])) and torch.equal(db[7:], torch.zeros_like(db[7:]))
    assert out.intact() and bias.intact(), (n, "sentinel after the output overwritten")
    if n >= 4173:
        print(f"\n[dw_exact] nm_dw_gemm n={n} trunk_only={trunk_only}: max |v - e| / B per item " +
              " ".join(f"{u:.2e}" for u in use))


def _T():
    return 128 * _sm()


AG_SIZES = [1, 65, 4173, "T+1", STEP]


@pytest.fixture(scope="module")
def nets():
    return kind_nets(DEV)


@pytest.mark.parametrize("kind", list(dx.KINDS))
@pytest.mark.parametrize("size", AG_SIZES)
def test_parameter_gradients_in_exact_windows(nets, kind, size, monkeypatch):
    """Joiner.forward under autograd, (raw * g).sum().backward(): the planes the step used are recorded by call-through
    wrappers of autograd._chain_kernel, _dw_kernel and _encodings, and every element of every parameter's .grad lies in
    param_windows (layout from the reference's module, windows of the engine that summed it)."""
    n = _T() + 1 if size == "T+1" else size
    j = nets[kind]
    rec = {}
    chain, dwk, enc = nag._chain_kernel, nag._dw_kernel, nag._encodings

    def chain_rec(joiner, P, stash, g):
        out = chain(joiner, P, stash, g)
        rec.update(stash=stash, g=g, chain=out)
        return out

    def dw_rec(ctx, g_pre, g_f, g_v, sx, sf, n_):
        rec['dw_calls'] = rec.get('dw_calls', 0) + 1
        return dwk(ctx, g_pre, g_f, g_v, sx, sf, n_)

    def enc_rec(joiner, pts, views):
        out = enc(joiner, pts, views)
        rec['enc'] = out
        return out
    monkeypatch.setattr(nag, "_chain_kernel", chain_rec)
    monkeypatch.setattr(nag, "_dw_kernel", dw_rec)
    monkeypatch.setattr(nag, "_encodings", enc_rec)
    gen = torch.Generator(device=DEV).manual_seed(n)
    pts, views = kind_inputs(kind, n, gen, DEV)
    g = torch.randn(n, 4, device=DEV, generator=gen)
    j.zero_grad()
    raw = nag.joiner_forward(j, pts, views)
    (raw * g).sum().backward()
    assert rec.get('dw_calls') == 1 and 'enc' in rec
    sx, sf, sv, _ = rec['stash']
    g_pre, g_f, g_v, inv = rec['chain']
    pe, dpe = rec['enc']
    planes = dict(g=rec['g'], g_pre=g_pre, g_f=g_f, g_v=g_v, sx=sx, sf=sf, sv=sv, pe=pe, dpe=dpe)
    win = dx.param_windows(kind, planes, float(inv))
    lines = []
    for name, p in j.nerf.named_parameters():
        e, B = win[name]
        v = p.grad.reshape(e.shape)
        dx.assert_in_window(f"{kind} n={n} {name}", v, e, B)
        lines.append(f"{name} {dx.used(v, e, B):.2e}")
    if n >= 4173:
        print(f"\n[dw_exact] {kind} n={n} max |v - e| / B: " + "; ".join(lines))


@pytest.mark.parametrize("n", [65, 4173])
def test_subnormal_operands(n):
    """The subnormal allowance of dw_window (dx.mma_abs) is needed where the gradient operand is an fp16 subnormal and
    nowhere else.  Gradient channel 0 of every plane holds subnormals (multiples of 2^-24), channel 1 the same values
    times 2^18 (normal): exact results differ by 2^18 exactly.  k_dw_gemm: channel 1 lies in the window WITHOUT the
    allowance, channel 0 in the window with it; the same for _wgrad (cuBLAS) against the order-free window.  On the adversarial planes (activation rows up to 60000 next to 1e-3 rows),
    where k_dw_gemm's subnormal channels needed the allowance; how much of it is printed."""
    planes = dx.dw_planes(n, 1000 + n, DEV)
    for key in ('g_pre', 'g_f', 'g_v'):
        t = planes[key].float()
        t[..., 0] = (t[..., 8].clamp(-2.0, 2.0) * 2.0 ** -18).half().float()        # channel 8: normal-sized values
        t[..., 1] = t[..., 0] * 2.0 ** 18
        planes[key] = t.half()
        assert float(planes[key][..., 0].float().abs().max()) < dx.MIN16
        assert float((planes[key][..., 0] != 0).float().mean()) > 0.2
    ctx = ops._ctx_for(planes['g_f'])
    dw = torch.empty(9, 256, 256, device=DEV)
    db = torch.empty(9, 256, device=DEV)
    ctx.check(ctx.lib.nm_dw_gemm(ctx.h, _p(planes['g_pre']), _p(planes['g_f']), _p(planes['g_v']), _p(planes['sx']),
                                 _p(planes['sf']), n, _p(dw), _p(db), ctx.stream()))
    worst_plain = worst_mm = 0.0
    for k, (G, X) in enumerate(dx.dw_items(planes)):
        e, B = dx.dw_window(G[:, :2], X)
        e0, B0 = dx.dw_window(G[:, :2], X, align_subnormals=False)
        v = dw[k, :2]
        dx.assert_in_window(f"item {k} normal channel, no allowance", v[1], e0[1], B0[1])
        dx.assert_in_window(f"item {k} subnormal channel", v[0], e[0], B[0])
        worst_plain = max(worst_plain, dx.used(v[0], e0[0], B0[0]))
        e, B = dx.gemm_window_any_order(G[:, :2], X)
        e0, B0 = dx.gemm_window_any_order(G[:, :2], X, align_subnormals=False)
        v = nag._wgrad(G[:, :2].contiguous(), X)
        dx.assert_in_window(f"item {k} _wgrad normal channel, no allowance", v[1], e0[1], B0[1])
        dx.assert_in_window(f"item {k} _wgrad subnormal channel", v[0], e[0], B[0])
        worst_mm = max(worst_mm, dx.used(v[0], e0[0], B0[0]))
    print(f"\n[dw_exact] n={n} subnormal channel: max |v - e| / B without the allowance: k_dw_gemm {worst_plain:.2f}, "
          f"_wgrad {worst_mm:.2f}")


@pytest.mark.parametrize("width", [64, 96])
def test_wgrad_split_keeps_fp32_accuracy(width):
    """_wgrad, the K = n GEMMs of the encodings and heads, in the order-free window at the sizes where a single cuBLAS
    GEMM with K = n reduced below fp32 on the H100 (n ~ 14 000 - 40 000; also T + 1 of this GPU and one training step).
    The single GEMM's use of its window is printed for comparison."""
    gen = torch.Generator(device=DEV).manual_seed(width)
    rows = []
    for n in (4097, 14593, 16897, 18433, 24577, 33793, _T() + 1, STEP):
        G = (torch.randn(n, 256, device=DEV, generator=gen) * (torch.rand(n, 256, device=DEV, generator=gen) < 0.5)).half()
        X = torch.randn(n, width, device=DEV, generator=gen).half()
        e, B = dx.gemm_window_any_order(G, X)
        v = nag._wgrad(G, X)
        dx.assert_in_window(f"_wgrad n={n} width={width}", v, e, B)
        rows.append(f"{n}: {dx.used(v, e, B):.1e} (one GEMM {dx.used(torch.mm(G.t(), X, out_dtype=torch.float32), e, B):.1e})")
    print(f"\n[dw_exact] _wgrad width {width} max |v - e| / B: " + "; ".join(rows))
