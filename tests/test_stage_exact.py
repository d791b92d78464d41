"""The exact restatements of tests/stage_exact.py against the oracle and the committed golden vectors (no GPU), and the
planted defects their checks must reject."""
import numpy as np
import pytest
import torch

from oracle import neuman_oracle as no
from oracle import synth_smpl
from tests import stage_exact as sx
from tests import util

F32 = np.float32


def test_raygen_restatement_matches_golden():
    g = util.golden("stages.npz")
    H, W = (int(v) for v in g["cam_HW"])
    o, d = sx.raygen(g["cam_K"], g["cam_c2w"], W, 0, xy=no.all_pixel_coords(H, W))
    assert np.array_equal(o, g["rays_o0"]) and np.abs(d - g["rays_d0"]).max() <= 1.2e-7     # numpy's summation order
    _, d1 = sx.raygen(g["cam_K"], g["cam_c2w"], W, 1, pix=np.arange(H * W))
    assert np.abs(d1 - g["rays_d1"]).max() <= 1.2e-7
    _, d2 = sx.raygen(g["cam_K"], g["cam_c2w"], W, 0, pix=np.arange(H * W))
    assert np.array_equal(d2, d)                     # pixel range == the same pixels as a list


def test_ray_to_samples_restatement_matches_torch():
    g = util.golden("stages.npz")
    S = g["s_z"].shape[1]
    o, d, n, f = (torch.from_numpy(g[k]) for k in ("s_o", "s_d", "s_near", "s_far"))
    for kw, ref in (({}, "s_z"), (dict(t_rand=g["s_trand"]), "s_z_perturb"), (dict(lindisp=True), "s_z_lindisp")):
        pts, z = sx.ray_to_samples(g["s_o"], g["s_d"], g["s_near"][:, 0], g["s_far"][:, 0], S, **kw)
        tk = dict(lindisp=kw.get("lindisp", False))
        if "t_rand" in kw:
            tk.update(perturb=1.0, t_rand=torch.from_numpy(g["s_trand"]))
        pt, _, zt = no.ray_to_samples(o, d, n, f, S, **tk)
        # torch's CPU kernels may contract a * b + c into an FMA, the restated kernel does not: one ulp apart at most
        assert (np.abs(z - zt.numpy()) <= 4 * np.spacing(np.abs(z))).all(), sx.first_diff(ref, z, zt.numpy())
        assert np.abs(pts - pt.numpy()).max() < 2e-6
        assert np.abs(z - g[ref]).max() < 2e-6


def _tangent_rays(verts, centres, radii, thr, origin_dist, rng, rel=(1e-4,), toward=None):
    """rays from cameras `origin_dist` away from the body passing at radius * (1 -+ rel) from each centre, on the side
    away from the body's middle"""
    mid = verts.mean(0)
    o_list, d_list = [], []
    for c, r in zip(centres, radii):
        cam = mid + rng.normal(size=3)
        cam = mid + (cam - mid) / np.linalg.norm(cam - mid) * origin_dist
        u = (c - cam) / np.linalg.norm(c - cam)
        a = (toward[len(o_list) // (2 * len(rel))] if toward is not None else mid) - c
        a = -a if toward is None else a
        out = a - (a @ u) * u
        out = out / max(np.linalg.norm(out), 1e-12) if np.linalg.norm(out) > 1e-9 else np.cross(u, [0, 0, 1.0])
        for s in [1 + sg * r_ for r_ in rel for sg in (-1, 1)]:
            tgt = c + out * (r * s)
            dd = tgt - cam
            o_list.append(cam)
            d_list.append(dd / np.linalg.norm(dd))
    return np.array(o_list, F32), np.array(d_list, F32)


def near_far_cases(seed=0, n_verts=None, dists=(1, 10, 50)):
    """(verts, origins, dirs, threshold): rays tangent to the outermost vertices' threshold spheres and to the groups'
    cull spheres, plus random rays, non-unit directions and origins inside the body"""
    rng = np.random.RandomState(seed)
    body = synth_smpl.random_body(seed=2, center=(0.1, 0.0, 0.3))
    V = body["verts"].astype(F32)
    if n_verts is not None:
        V = V[rng.choice(V.shape[0], n_verts, replace=False)]
    thr = float(body["geo_threshold"])
    gv, gc, gr, bc, br = sx.vertex_groups(V)
    far_v = np.argsort(-np.linalg.norm(V - bc, axis=1))[:8]
    os_, ds_ = [], []
    for k, D in enumerate(dists):
        Dw = D * float(br)
        o, d = _tangent_rays(V, V[far_v], np.full(len(far_v), thr), thr, Dw, rng)
        os_.append(o); ds_.append(d)
        pick = rng.choice(len(gc), min(len(gc), 24), replace=False)
        far_g = gv[pick, np.argmax(((gv[pick] - gc[pick][:, None]) ** 2).sum(-1), 1)]
        o, d = _tangent_rays(V, gc[pick], gr[pick] + F32(thr), thr, Dw, rng, rel=(1e-4, 3e-7, 1e-7, 0.0), toward=far_g)
        os_.append(o); ds_.append(d)
        cam = bc + rng.normal(size=(64, 3)) * Dw / np.sqrt(3)
        tgt = V[rng.randint(0, len(V), 64)] + rng.normal(0, thr, (64, 3))
        dd = tgt - cam
        os_.append(cam.astype(F32)); ds_.append((dd / np.linalg.norm(dd, axis=1, keepdims=True)).astype(F32))
    inside = V[rng.randint(0, len(V), 32)] + rng.normal(0, 0.02, (32, 3))
    os_.append(inside.astype(F32)); ds_.append(rng.normal(size=(32, 3)).astype(F32))     # non-unit directions
    return V, np.concatenate(os_), np.concatenate(ds_), thr


def test_near_far_restatements_agree_and_match_oracle():
    for n_verts in (None, 17, 65):                       # SMPL-sized, < 32 vertices, n_verts = 1 (mod 32)
        V, o, d, thr = near_far_cases(n_verts=n_verts)
        n0, f0 = sx.near_far_exhaustive(o, d, V, thr)
        n1, f1 = sx.near_far_groups(o, d, V, thr)
        n2, f2 = sx.near_far_body_cull(o, d, V, thr)
        for name, a, b in (("groups near", n1, n0), ("groups far", f1, f0), ("body near", n2, n0), ("body far", f2, f0)):
            assert np.array_equal(a, b), sx.first_diff(name, a, b)
        hit = np.isfinite(n0)
        assert 0.2 < hit.mean() < 0.95, hit.mean()
    # the exhaustive restatement is the oracle's formula: the committed reference near/far to rounding
    g = util.golden("stages.npz")
    body = synth_smpl.random_body(seed=2, center=(0.1, 0.0, 0.3))
    n, f = sx.near_far_exhaustive(g["nf_o"], g["nf_d"], body["verts"], float(g["nf_thr"]))
    hit = ~np.isinf(g["nf_near"])
    solid = hit & ((g["nf_far"] - g["nf_near"]) > 1e-3)
    assert np.abs(n[solid] - g["nf_near"][solid]).max() < 3e-5 and np.abs(f[solid] - g["nf_far"][solid]).max() < 3e-5
    assert (n[~hit] == np.inf).all() and (f[~hit] == -np.inf).all()


def test_cdf_restatement_matches_torch():
    """build_cdf / invert_cdf against torch's cumsum and searchsorted: the cdf within 2 ulp of torch's (both accumulate
    in double, in different orders), and every sample that differs by more than rounding sits on the den < 1e-5 rule
    with den within rounding of 1e-5."""
    g = util.golden("stages.npz")
    rng = np.random.RandomState(1)
    w = (rng.rand(40, 300) ** 6).astype(F32)
    w[::7] = 0
    for W in (g["p_w"], w):
        t = torch.from_numpy(W) + 1e-5
        cdf_t = torch.cat([torch.zeros(W.shape[0], 1), torch.cumsum(t / t.sum(-1, keepdim=True), -1)], -1).numpy()
        cdf = sx.build_cdf(W)
        close = np.abs(cdf - cdf_t) <= 2 * np.spacing(np.maximum(cdf, cdf_t).astype(F32))
        assert close.all(), sx.first_diff("cdf", cdf, cdf_t)
    out = sx.sample_pdf(g["p_bins"], g["p_w"], 11, u=g["p_u"])
    _, den = sx.invert_cdf(sx.build_cdf(g["p_w"]), g["p_bins"], g["p_u"], with_den=True)
    # torch may contract the interpolation into FMAs: a few ulp; anything more must be the 1e-5 rule
    diff = np.abs(out - g["p_out"]) > 2e-6
    named = [tuple(int(k) for k in i) for i in np.argwhere(diff)]
    assert all(abs(float(den[i]) - 1e-5) < 1e-9 for i in named), [(i, float(den[i])) for i in named]
    print("samples on the 1e-5 discontinuity:", named)
    assert np.abs(out - g["p_out"])[~diff].max() <= 2e-6


def test_importance_restatement_matches_oracle():
    torch.manual_seed(5)
    R, S, N = 64, 64, 128
    o, d = torch.randn(R, 3), torch.nn.functional.normalize(torch.randn(R, 3), dim=-1)
    _, _, z = no.ray_to_samples(o, d, torch.zeros(R, 1), torch.full((R, 1), 3.14), S)
    w = torch.rand(R, S) ** 6
    for inc in (True, False):
        _, _, zt = no.ray_to_importance_samples(o, d, z, w, N, including_old=inc)
        _, zs = sx.importance(o.numpy(), d.numpy(), z.numpy(), w.numpy(), N, including_old=inc)
        bad = np.abs(zs - zt.numpy()) > 2e-6
        # differences only where torch's cdf sits on the other side of the 1e-5 rule: at most one bin
        assert bad.mean() < 0.02 and np.abs(zs - zt.numpy()).max() <= 3.14 / (S - 1) * 1.01


def test_merge_restatement_is_the_stable_sort():
    rng = np.random.RandomState(2)
    zs = [np.sort(rng.rand(9, s).astype(F32), 1) for s in (5, 7, 3)]
    zs[1][:, 2] = zs[0][:, 1]
    raws = [rng.randn(9, z.shape[1], 4).astype(F32) for z in zs]
    z, r = sx.merge(zs, raws)
    zt, order = torch.sort(torch.from_numpy(np.concatenate(zs, 1)), dim=-1, stable=True)
    assert np.array_equal(z, zt.numpy())
    assert np.array_equal(r, np.take_along_axis(np.concatenate(raws, 1), order.numpy()[..., None], 1))


def _composite_inputs(seed, R, S, opaque=True):
    rng = np.random.RandomState(seed)
    z = np.sort(rng.uniform(2, 6, (R, S)), 1).astype(F32)
    raw = (rng.randn(R, S, 4) * 1.5).astype(F32)
    d = rng.randn(R, 3).astype(F32)
    if opaque:
        s = rng.randint(0, S, R)
        dist = np.where(s + 1 < S, z[np.arange(R), np.minimum(s + 1, S - 1)] - z[np.arange(R), s], 1.0)
        raw[np.arange(R), s, 3] = rng.uniform(5, 40, R) / np.maximum(dist * np.linalg.norm(d, axis=1), 1e-6)
    return raw, z, d


def test_composite_reference_is_autograd_in_float64():
    """The exact values of the windows are torch's raw2outputs and its autograd gradient in float64, on inputs whose
    fp32 prefix (distances, sigma * dist) is exact.  The windows start from the fp32 alpha (stage_exact._alpha_f), so the
    two agree to that rounding."""
    rng = np.random.RandomState(3)
    R, S = 6, 40
    z = np.cumsum(rng.randint(1, 8, (R, S)) / 64.0, 1).astype(F32)
    raw = rng.randn(R, S, 4).astype(F32)
    raw[..., 3] = rng.randint(-16, 64, (R, S)) / 4.0
    d = np.tile(np.array([[0, 0, 1]], F32), (R, 1))
    g = [rng.randn(R, 3).astype(F32), rng.randn(R).astype(F32), rng.randn(R).astype(F32), rng.randn(R, S).astype(F32)]
    fw = sx.composite_forward(raw, z, d, white_bkg=True)
    bw = sx.composite_backward(raw, z, d, *g, white_bkg=True)
    rt = torch.from_numpy(raw).double().requires_grad_(True)
    with no.precision(torch.float64):
        rgb, disp, acc, w, depth = no.raw2outputs(rt, torch.from_numpy(z).double(), torch.from_numpy(d).double(), white_bkg=True)
    (rgb * torch.from_numpy(g[0])).sum().add((depth * torch.from_numpy(g[1])).sum()).add(
        (acc * torch.from_numpy(g[2])).sum()).add((w * torch.from_numpy(g[3])).sum()).backward()
    for name, t in (("w", w), ("rgb", rgb), ("acc", acc), ("depth", depth)):
        assert np.allclose(fw[name].e, t.detach().numpy(), rtol=1e-5, atol=1e-7), name
    assert np.allclose(bw.e, rt.grad.numpy(), rtol=1e-5, atol=1e-6)


def test_composite_windows_hold_the_fp32_chain():
    """The float32 emulation of both kernels (numpy's expf, the kernels' order) lies inside the windows."""
    for S in (1, 2, 31, 33, 96):
        raw, z, d = _composite_inputs(S, 12, S)
        noise = np.random.RandomState(S).randn(12, S).astype(F32) * 0.5
        for wb in (True, False):
            fw = sx.composite_forward(raw, z, d, noise=noise, sigma_scale=0.7, white_bkg=wb)
            for k, v in fw.items():
                assert sx.outside(k, v.f, v) is None, sx.outside(k, v.f, v)
            g = np.random.RandomState(1).randn(12, 3).astype(F32)
            bw = sx.composite_backward(raw, z, d, g_rgb=g, g_depth=g[:, 0], g_acc=g[:, 1], g_w=raw[..., 0], noise=noise,
                                       sigma_scale=0.7, white_bkg=wb)
            assert sx.outside("d_raw", bw.f, bw) is None, sx.outside("d_raw", bw.f, bw)


# ---------------------------------------------------------------------------------------------
# planted defects
# ---------------------------------------------------------------------------------------------
DEFECTS = ["searchsorted_left", "dropped_carry", "cancelling_suffix", "unstable_merge"]


@pytest.mark.parametrize("defect", DEFECTS)
def test_rule_rejects_planted_defects(defect):
    if defect in ("searchsorted_left", "dropped_carry"):
        rng = np.random.RandomState(4)
        R, B, N = 16, 100, 256
        bins = np.sort(rng.rand(R, B).astype(F32), 1)
        w = (rng.rand(R, B - 1) ** 4).astype(F32)
        cdf = sx.build_cdf(w)
        u = np.concatenate([cdf[:, ::3], np.zeros((R, 1), F32), np.full((R, 1), cdf[0, -1], F32),
                            rng.rand(R, N).astype(F32)], 1)            # u exactly on cdf entries, 0 and cdf[-1]
        good = sx.sample_pdf(bins, w, u.shape[1], u=u)
        bad = sx.sample_pdf(bins, w, u.shape[1], u=u, **({"right": False} if defect == "searchsorted_left" else
                                                          {"drop_carry": True}))
        msg = sx.first_diff("sample_pdf", bad, good)
    elif defect == "cancelling_suffix":
        raw, z, d = _composite_inputs(7, 8, 64)
        g = np.random.RandomState(8).randn(8, 3).astype(F32)
        window = sx.composite_backward(raw, z, d, g_rgb=g)
        bad = sx.composite_backward(raw, z, d, g_rgb=g, suffix="subtract")
        msg = sx.outside("d sigma", bad.f[..., 3], window[..., 3])
    else:
        rng = np.random.RandomState(5)
        zs = [np.round(rng.rand(4, s) * 8).astype(F32) / 8 for s in (6, 5)]     # many exact ties
        raws = [rng.randn(4, z.shape[1], 4).astype(F32) for z in zs]
        good = sx.merge(zs, raws)[1]
        bad = sx.merge(zs, raws, stable=False)[1]
        msg = sx.first_diff("raw", bad, good)
    print(defect, "->", msg)
    assert msg is not None, f"{defect} was not rejected"
