"""The exact-window rule of tests/dw_exact.py, checked on the CPU.

k_dw_gemm: numpy fp32 emulations of the kernel's summation (16-row MMAs over random contiguous 64-row CTA ranges, the
partials reduced in random order), a pairwise fp32 sum and the float64 sum rounded once are accepted on every element,
on plain and on adversarial planes; each planted defect of the kind a pipeline or work-list rewrite can introduce is
rejected at the sizes tests/test_gpu_dw_exact.py launches.

The assembly: param_windows, written from the reference's module, equals torch autograd's parameter gradients of a
float64 forward of the fp16-quantised net for every net kind; neuman_b200.autograd._weight_grads itself, run on the CPU
on the same planes (float64 GEMMs in place of the kernels), lies in those windows; and planted assembly defects
(encoding columns out of order, a bias from the wrong column, the halves of views_linears.0 swapped, a head on the wrong
layer) are rejected."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import dw_exact as dx
from tests import tc_exact as tx
from tests import util

SIZES = (1, 63, 64, 65, 4173, 14213)
PAIRS = 66                                        # CTA pairs of an H100 SXM (132 SMs): the GPU test's partition sizes
GPU_SIZES = (1, 63, 64, 65, 640, 64 * PAIRS - 1, 64 * PAIRS + 1, 2 * 64 * PAIRS - 1, 2 * 64 * PAIRS + 1, 4173, 14213,
             2048 * 128 + 77)
W, V = 32, 16                                     # plane widths here (the windows do not depend on them)


# ---------------------------------------------------------------------------------------------
# numpy fp32 emulations of one k_dw_gemm work item
# ---------------------------------------------------------------------------------------------
def _np(t):
    return t.numpy() if isinstance(t, torch.Tensor) else t


def block_products(G, X):
    """fp32 [ceil(n/16), M, N]: each 16-row MMA's G^T X (fp32 matmul of the fp16 operands, rows past n zero)."""
    G = _np(G).astype(np.float32)
    X = np.ones((G.shape[0], 1), np.float32) if X is None else _np(X).astype(np.float32)
    n = G.shape[0]
    pad = -n % 16
    G = np.concatenate([G, np.zeros((pad, G.shape[1]), np.float32)])
    X = np.concatenate([X, np.zeros((pad, X.shape[1]), np.float32)])
    k = G.shape[0] // 16
    return np.matmul(G.reshape(k, 16, -1).transpose(0, 2, 1), X.reshape(k, 16, -1)).astype(np.float32)


def cta_partials(P, cuts, defect=None, target=None):
    """One fp32 partial per CTA: CTA c runs the 16-row MMAs of rows [cuts[c], cuts[c + 1]) in ascending order (a
    sequential fp32 accumulation).  Defects: 'stage_dropped' skips one 64-row stage of CTA `target`, 'stale_slot' makes
    one of its stages re-read the rows of the stage DW_STAGES earlier (what a consumer reads from a ring slot that was not
    refilled), 'tail_dropped' skips the rows past the last multiple of 64."""
    n_blocks = P.shape[0]
    out = []
    for c in range(len(cuts) - 1):
        b0, b1 = cuts[c] // 16, min(n_blocks, -(-cuts[c + 1] // 16))
        idx = list(range(b0, b1))
        if c == target and defect in ("stage_dropped", "stale_slot"):
            stages = [idx[i:i + 4] for i in range(0, len(idx), 4)]
            s = len(stages) // 2
            if defect == "stage_dropped":
                stages[s] = []
            elif len(stages) > dx.DW_STAGES:                                  # the ring wraps only past DW_STAGES
                s = max(s, dx.DW_STAGES)
                stages[s] = [b - 4 * dx.DW_STAGES for b in stages[s]]
            idx = [b for st in stages for b in st]
        if defect == "tail_dropped":
            idx = [b for b in idx if 16 * b < cuts[-1] // 64 * 64]
        acc = np.cumsum(P[idx], axis=0, dtype=np.float32)[-1] if idx else np.zeros(P.shape[1:], np.float32)
        out.append(acc)
    return out


def reduce_partials(parts, order):
    acc = np.zeros_like(parts[0])
    for i in order:
        acc = (acc + parts[i]).astype(np.float32)
    return acc


def random_cuts(n, rng, n_parts=None):
    """Contiguous CTA row ranges: boundaries on multiples of 64, the last one n."""
    blocks = -(-n // 64)
    p = n_parts or int(rng.integers(1, dx.n_parts_max(n) + 1))
    p = min(p, blocks)
    inner = np.sort(rng.choice(np.arange(1, blocks), size=p - 1, replace=False)) if p > 1 else np.array([], int)
    return [0] + [int(b) * 64 for b in inner] + [n]


def even_cuts(n, p):
    blocks = -(-n // 64)
    p = min(p, blocks)
    return [min(n, blocks * i // p * 64) for i in range(p)] + [n]


def emulate_kernel(P, n, rng):
    cuts = random_cuts(n, rng)
    parts = cta_partials(P, cuts)
    return reduce_partials(parts, rng.permutation(len(parts)))


def emulate_pairwise(G, X):
    """fp32 pairwise tree over the exact per-row products."""
    G = _np(G).astype(np.float32)
    X = np.ones((G.shape[0], 1), np.float32) if X is None else _np(X).astype(np.float32)
    t = G[:, :, None] * X[:, None, :]                           # fp16 x fp16 products are exact in fp32
    while t.shape[0] > 1:
        if t.shape[0] % 2:
            t = np.concatenate([t, np.zeros_like(t[:1])])
        t = (t[0::2] + t[1::2]).astype(np.float32)
    return t[0]


def emulate_f64(G, X):
    G = _np(G).astype(np.float64)
    X = np.ones((G.shape[0], 1)) if X is None else _np(X).astype(np.float64)
    return (G.T @ X).astype(np.float32)


def _check(name, v, e, B):
    return tx.check32(name, torch.from_numpy(np.asarray(v)), e, B)


@pytest.mark.parametrize("adversarial", [False, True])
@pytest.mark.parametrize("n", SIZES)
def test_rule_accepts_fp32_evaluations(n, adversarial):
    """Every element of every work item's dW and bias gradient, evaluated in fp32 in three kernel-like orders (random
    CTA ranges and reduction orders), pairwise, and as the float64 sum rounded once, lies in its window."""
    planes = dx.dw_planes(n, 100 + n, "cpu", width=W, views=V, adversarial=adversarial)
    rng = np.random.default_rng(n)
    for k, (G, X) in enumerate(dx.dw_items(planes)):
        for x, tag in ((X, "dw"), (None, "db")):
            e, B = dx.dw_window(G, x)
            P = block_products(G, x)
            evals = [emulate_kernel(P, n, rng) for _ in range(3)] + [emulate_pairwise(G, x), emulate_f64(G, x)]
            for i, v in enumerate(evals):
                c = _check(f"item {k} {tag} evaluation {i}", v, e, B)
                assert c.ok.all(), (n, adversarial, c.message())


def test_adversarial_planes_are_adversarial():
    """The adversarial planes hold what the rule is meant to face: +-60000 next to 1e-3, fp16 subnormal gradients,
    all-zero rows, exactly cancelling row pairs."""
    p = dx.dw_planes(4173, 7, "cpu", width=W, views=V)
    G, X = p['g_pre'][3].double(), p['sx'][2].double()
    assert float(G.abs().max()) >= 59000 and float(X.abs().max()) >= 20000
    nz = G.abs()[G != 0]
    assert float(nz.min()) < 2.0 ** -14                                   # fp16 subnormals
    assert bool(((G == 0).all(1)).any())
    cancel = (G[1:] == -G[:-1]).all(1) & (X[1:] == X[:-1]).all(1) & (G[1:] != 0).any(1)
    assert int(cancel.sum()) > 100
    sub = G[:, :4].abs()                                                  # channels that hold nothing but subnormals
    assert float(sub.max()) < 2.0 ** -14 and bool((sub > 0).any())


DEFECTS = ("stage_dropped", "stale_slot", "tail_dropped", "half_missing", "half_twice", "partials_f16", "items_swapped",
           "bias_from_x")


def _defective(planes, n, defect, rng):
    """(dw [items, M, N], db [items, M]) of the whole launch with one planted defect, on a host-like split into
    up to 8 CTAs per item (what an H100's 66 CTA pairs give each of the nine items)."""
    items = dx.dw_items(planes)
    dws, dbs = [], []
    for k, (G, X) in enumerate(items):
        cuts = even_cuts(n, 8)
        order = rng.permutation(len(cuts) - 1)
        target = int(np.argmax(np.diff(cuts)))                            # the CTA with the most stages
        out = []
        for x in (X, None):
            P = block_products(G, x)
            kw = dict(defect=defect, target=target) if (k == 0 and defect in ("stage_dropped", "stale_slot")) else {}
            if defect == "tail_dropped":
                kw = dict(defect=defect)
            parts = cta_partials(P, cuts, **kw)
            if defect == "partials_f16":
                parts = [p.astype(np.float16).astype(np.float32) for p in parts]
            if k == 0 and defect in ("half_missing", "half_twice"):              # the CTA of output rows [M/2, M)
                h = parts[target].shape[0] // 2
                half = parts[target].copy()
                half[:h] = 0
                if defect == "half_missing":
                    parts[target] = parts[target] - half
                else:
                    parts.append(half)
            out.append(reduce_partials(parts, list(order) + list(range(len(order), len(parts)))))
        dws.append(out[0])
        dbs.append(out[1][:, 0])
    if defect == "items_swapped":
        dws[0], dws[1] = dws[1], dws[0]
    if defect == "bias_from_x":
        dbs[0] = emulate_f64(items[0][1], None)[:, 0][:items[0][0].shape[1]]
    return dws, dbs


_CASES = {}


def _case(n):
    """plain planes of n rows, the windows of every item, and the defect-free emulation"""
    if n not in _CASES:
        planes = dx.dw_planes(n, 200 + n, "cpu", width=W, views=V, adversarial=False)
        wins = []
        for G, X in dx.dw_items(planes):
            e, B = dx.dw_window(G, X)
            eb, Bb = dx.dw_window(G, None)
            wins.append(((e, B), (eb[:, 0], Bb[:, 0])))
        _CASES[n] = (planes, wins, _defective(planes, n, None, np.random.default_rng(n)))
    return _CASES[n]


@pytest.mark.parametrize("defect", DEFECTS)
def test_rule_rejects_planted_kernel_defects(defect):
    """Each structural defect (rows lost, re-read or counted twice, outputs misplaced) is rejected on at least one
    element at every size of the GPU test where it changes the result.  Partials rounded to fp16 move an element by at
    most 2^-12 of a partial, which the MMA term of the window exceeds once a CTA runs more than ~30 instructions: that
    defect is rejected at the small sizes only.  The rejected fraction of the changed elements is printed per size."""
    report = []
    for n in GPU_SIZES:
        planes, wins, (good_w, good_b) = _case(n)
        dws, dbs = _defective(planes, n, defect, np.random.default_rng(n))
        changed = rejected = 0
        for k in range(len(wins)):
            for v, good, (e, B) in ((dws[k], good_w[k], wins[k][0]), (dbs[k], good_b[k], wins[k][1])):
                c = _check(f"item {k}", v, e, B)
                ch = torch.from_numpy(np.asarray(v) != good)
                changed += int(ch.sum())
                rejected += int((~c.ok & ch).sum())
        if changed:
            report.append((n, rejected, changed))
            assert rejected > 0 or defect == "partials_f16", (defect, n, "changes", changed, "elements, none rejected")
    assert report and max(r for _, r, _ in report) > 0, (defect, "never rejected")
    print(f"\n[dw_exact] {defect}: rejected / changed elements per n: " +
          ", ".join(f"{n}: {r}/{c} ({r / c:.3f})" for n, r, c in report))


# ---------------------------------------------------------------------------------------------
# The assembly: param_windows against float64 autograd, and _weight_grads run on the CPU
# ---------------------------------------------------------------------------------------------
def kind_nets(device="cpu"):
    """One Joiner of every kind param_windows knows."""
    import neuman_b200 as nb
    from tests import nerft_cases, viewless_cases
    from tests.test_tc_exact import carrier_joiner
    coarse, _, human = util.product_nets(device)
    carrier = carrier_joiner().to(device)
    for p in carrier.nerf.parameters():
        p.requires_grad_(True)
    return {"posenc": coarse, "rotate": human, "carrier": carrier,
            "nerft": nerft_cases.nerft_nets(nb.build_nerf, nb.default_opt)[0].to(device),
            "viewless": viewless_cases.viewless_nets(nb.build_nerf, nb.default_opt, "posenc")[0].to(device)}


def kind_inputs(kind, n, gen, device):
    """(pts, views) of n samples: NeRF-T with one time per ray of 128 samples, the carrier with zero views (as
    models.offset_forward_at_time passes them), views None for a view-independent net."""
    pts = torch.randn(n, 3, generator=gen, device=device) * 1.5
    views = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen, device=device), dim=-1)
    if kind == "nerft":
        t = torch.rand(-(-n // 128), generator=gen, device=device).repeat_interleave(128)[:n]
        pts = torch.cat([pts, t[:, None]], 1)
    if kind == "carrier":
        views = torch.zeros_like(views)
    return pts, (None if kind == "viewless" else views)


class _Q16(torch.autograd.Function):
    """round to fp16 in the forward, identity in the backward (float64)"""
    @staticmethod
    def forward(ctx, x):
        return x.half().double()

    @staticmethod
    def backward(ctx, gy):
        return gy


def f64_step(j, pts, views, g, S):
    """A float64 forward of the reference's module (models/vanilla.py:120-152) on fp16-rounded operands -- every
    nn.Linear reads the fp16 tensor the kernels stash, the weights are rounded like the packed slabs -- and torch
    autograd of (raw * g).sum().  -> (planes as the training step records them, with the gradient planes exact and
    scaled by S; {parameter: float64 gradient})."""
    q = _Q16.apply
    P = {k: v.detach().double().clone().requires_grad_(True) for k, v in j.nerf.state_dict().items()}
    viewless = views is None
    pe = q(tx.embed64(pts, j.pos_pe))
    h, pres, sx = pe, [], []
    for l in range(8):
        pre = F.linear(h, q(P[f'pts_linears.{l}.weight']), P[f'pts_linears.{l}.bias'])
        pre.retain_grad()
        pres.append(pre)
        sx.append(q(torch.relu(pre)))
        h = torch.cat([pe, sx[-1]], -1) if l == 4 else sx[-1]
    if viewless:
        raw = F.linear(h, q(P['output_linear.weight']), P['output_linear.bias'])
    else:
        ve = q(tx.embed64(views, j.dir_pe))
        alpha = F.linear(h, q(P['alpha_linear.weight']), P['alpha_linear.bias'])
        feat = F.linear(h, q(P['feature_linear.weight']), P['feature_linear.bias'])
        feat.retain_grad()
        sf = q(feat)
        prev = F.linear(torch.cat([sf, ve], -1), q(P['views_linears.0.weight']), P['views_linears.0.bias'])
        prev.retain_grad()
        sv = q(torch.relu(prev))
        raw = torch.cat([F.linear(sv, q(P['rgb_linear.weight']), P['rgb_linear.bias']), alpha], -1)
    (raw * g.double()).sum().backward()
    n, n_pe = pts.shape[0], pe.shape[1]
    pe_plane = torch.zeros(n, 96 if n_pe > 63 else 64, dtype=torch.float64)       # nm_encode_f16's planes
    pe_plane[:, :n_pe], pe_plane[:, n_pe] = pe.detach(), 1.0
    planes = dict(g=g, g_pre=torch.stack([S * p.grad for p in pres]), sx=torch.stack([s.detach() for s in sx]), pe=pe_plane,
                  g_f=None, g_v=None, sf=None, sv=None, dpe=None)
    if not viewless:
        dpe = torch.zeros(n, 32, dtype=torch.float64)
        dpe[:, :ve.shape[1]], dpe[:, ve.shape[1]] = ve.detach(), 1.0
        planes.update(g_f=S * feat.grad, g_v=S * prev.grad, sf=sf.detach(), sv=sv.detach(), dpe=dpe)
    return planes, {k: p.grad for k, p in P.items()}


def _dw_f64(ctx, g_pre, g_f, g_v, sx, sf, n):
    """k_dw_gemm restated in float64, rounded to fp32 once"""
    dw = torch.zeros(9, 256, 256, dtype=torch.float64)
    db = torch.zeros(9, 256, dtype=torch.float64)
    for k in range(7):
        dw[k], db[k] = g_pre[k + 1].double().T @ sx[k].double(), g_pre[k + 1].double().sum(0)
    if g_f is not None:
        dw[7], db[7] = g_f.double().T @ sx[7].double(), g_f.double().sum(0)
        dw[8, :128], db[8, :128] = g_v.double().T @ sf.double(), g_v.double().sum(0)
    return dw.float(), db.float()


def assemble(monkeypatch, j, planes, inv, pe=None):
    """neuman_b200.autograd._weight_grads on the CPU: its two engines (k_dw_gemm, cuBLAS) replaced by float64 GEMMs
    rounded once, its encodings by the recorded planes (or `pe`); _wgrad's K blocks cut to 64 rows so that its split
    into whole blocks and a ragged rest is exercised."""
    from neuman_b200 import autograd as nag
    monkeypatch.setattr(nag, "_ctx_for", lambda t: None)
    monkeypatch.setattr(nag, "_mm32", lambda a, b: (a.double() @ b.double()).float())
    monkeypatch.setattr(nag, "_bmm32", lambda a, b: torch.bmm(a.double(), b.double()).float())
    monkeypatch.setattr(nag, "_K_CHUNK", 64)
    monkeypatch.setattr(nag, "_dw_kernel", _dw_f64)
    monkeypatch.setattr(nag, "_encodings", lambda joiner, p, v: (planes['pe'] if pe is None else pe, planes['dpe']))
    stash = (planes['sx'], planes['sf'], planes['sv'], None)
    return nag._weight_grads(j, stash, None, None, planes['g'], planes['g_pre'], planes['g_f'], planes['g_v'],
                             torch.tensor([inv], dtype=torch.float32))


def _sin_cos_swapped(j, pe):
    """the position plane with the sin and cos channels of the first frequency exchanged"""
    d, pe = j.pos_pe.input_dims, pe.clone()
    if j.pos_pe.mapping == 'rotate':
        nf = 3 * j.pos_pe.N_freqs
        a, b = slice(3, 3 + nf), slice(3 + nf, 3 + 2 * nf)
    else:
        a, b = slice(d, 2 * d), slice(2 * d, 3 * d)
    pe[:, a], pe[:, b] = pe[:, b].clone(), pe[:, a].clone()
    return pe


def _time_permuted(pe):
    """a NeRF-T position plane whose 21 time channels (t, sin f_k t, cos f_k t) are rotated by one"""
    cols = [3] + [c for k in range(10) for c in (7 + 8 * k, 11 + 8 * k)]
    pe = pe.clone()
    pe[:, cols] = pe[:, cols[1:] + cols[:1]]
    return pe


def _assembly_defects(kind, j, planes, inv, v, monkeypatch):
    """{defect: (the parameters it touches, the defective gradients)}"""
    n_pe = dx.KINDS[kind][0]
    out = {"sin_cos_swapped": (("pts_linears.0.weight", "pts_linears.5.weight"),
                               assemble(monkeypatch, j, planes, inv, pe=_sin_cos_swapped(j, planes['pe'])))}
    bad = dict(v)
    bad['pts_linears.0.bias'] = v['pts_linears.0.weight'][:, n_pe - 1]
    out["bias0_from_last_encoding_column"] = (("pts_linears.0.bias",), bad)
    if kind == "nerft":
        out["nerft_time_permuted"] = (("pts_linears.0.weight", "pts_linears.5.weight"),
                                      assemble(monkeypatch, j, planes, inv, pe=_time_permuted(planes['pe'])))
    head = "output_linear.weight" if kind == "viewless" else "alpha_linear.weight"
    cols = slice(0, 4) if kind == "viewless" else slice(3, 4)
    bad = dict(v)
    bad[head] = ((tx.r16(planes['g'].double() / inv)[:, cols].T @ planes['sx'][6].double()) * inv).float()
    out["head_from_sx6"] = ((head,), bad)
    if kind != "viewless":
        bad = dict(v)
        w = v['views_linears.0.weight']
        bad['views_linears.0.weight'] = torch.cat([w[:, 256:], w[:, :256]], 1)
        out["views_halves_swapped"] = (("views_linears.0.weight",), bad)
    return out


@pytest.mark.parametrize("kind", list(dx.KINDS))
def test_param_windows_pin_the_layout(kind, monkeypatch):
    """(1) param_windows' e equals torch autograd's parameter gradients of a float64 forward of the fp16-quantised net
    to 1e-12 (relative to each parameter's largest gradient); (2) _weight_grads on the same planes lies in the windows
    on every element; (3) each planted assembly defect leaves the window of the parameter it touches."""
    j = kind_nets()[kind]
    n = 333
    gen = torch.Generator().manual_seed(17)
    pts, views = kind_inputs(kind, n, gen, "cpu")
    g = torch.randn(n, 4, generator=gen).half().float()           # fp16 values: r16(g S) = g S exactly
    from neuman_b200.autograd import _pow2_scale
    S = float(_pow2_scale(g, 256.0))
    planes, ref = f64_step(j, pts, views, g, S)
    win = dx.param_windows(kind, planes, 1.0 / S)
    names = [k for k, _ in j.nerf.named_parameters()]
    assert sorted(win) == sorted(names)
    for k in names:
        e, B = win[k]
        assert e.shape == ref[k].shape, (k, e.shape, ref[k].shape)
        err = float((e - ref[k]).abs().max())
        assert err <= 1e-12 * float(ref[k].abs().max()), (kind, k, err)
    v = assemble(monkeypatch, j, planes, 1.0 / S)
    for k in names:
        c = tx.check32(k, v[k].reshape(win[k][0].shape), *win[k])
        assert c.ok.all(), (kind, c.message())
    for defect, (touched, bad) in _assembly_defects(kind, j, planes, 1.0 / S, v, monkeypatch).items():
        fr = []
        for k in touched:
            c = tx.check32(k, bad[k].reshape(win[k][0].shape), *win[k])
            fr.append(1.0 - float(c.ok.double().mean()))
        print(f"\n[dw_exact] {kind} {defect}: rejected fraction " + ", ".join(f"{k} {f:.3f}" for k, f in zip(touched, fr)))
        assert max(fr) > 0, (kind, defect, "accepted")
