"""The ray-marching stage kernels element by element against tests/stage_exact.py: bit-exact where the kernel uses only
correctly rounded operations, inside per-element float64 windows for the composite.  Each failure names the first
(ray, sample) outside."""
import ctypes as C

import numpy as np
import pytest
import torch

import neuman_b200 as nb
from neuman_b200 import ops
from neuman_b200._lib import Context, NmCamera
from oracle import scenes
from tests import stage_exact as sx
from tests.test_stage_exact import _composite_inputs, near_far_cases

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32 = np.float32


def cu(x):
    return torch.as_tensor(np.ascontiguousarray(x)).to(DEV)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def ctx():
    return Context.get(torch.cuda.current_device())


def exact(name, got, want):
    msg = sx.first_diff(name, got.cpu().numpy() if isinstance(got, torch.Tensor) else got, want)
    assert msg is None, msg


def test_raygen_bit_exact():
    c = ctx()
    for H, W, skew in ((17, 23, 0.0), (12, 40, 3.5)):
        K, c2w = scenes.camera(H, W, focal=40.0, seed=3)
        K = np.array(K, np.float64)
        K[0, 1] = skew
        K[1, 1] *= 1.37                                           # non-square pixels
        cap = nb.SimpleCapture(K, c2w, H, W)
        cam = ops.camera_struct(cap)
        for mode in (0, 1):
            for pix0, n in ((0, H * W), (5, 31)):
                o, d = torch.empty(n, 3, device=DEV), torch.empty(n, 3, device=DEV)
                c.check(c.lib.nm_raygen(c.h, C.byref(cam), mode, pix0, n, None, _p(o), _p(d), c.stream()))
                ro, rd = sx.raygen(K, cap.cam_pose.camera_to_world, W, mode, pix=np.arange(pix0, pix0 + n))
                exact(f"raygen origins mode {mode}", o, ro)
                exact(f"raygen dirs mode {mode} {H}x{W}", d, rd)
            xy = np.stack([np.random.RandomState(1).randint(-3, W + 3, 77), np.random.RandomState(2).randint(-3, H + 3, 77)], 1)
            xyt = cu(xy.astype(np.int32))
            o, d = torch.empty(77, 3, device=DEV), torch.empty(77, 3, device=DEV)
            c.check(c.lib.nm_raygen(c.h, C.byref(cam), mode, 0, 77, _p(xyt), _p(o), _p(d), c.stream()))
            exact(f"raygen xy dirs mode {mode}", d, sx.raygen(K, cap.cam_pose.camera_to_world, W, mode, xy=xy)[1])


@pytest.mark.parametrize("S", [1, 2, 3, 31, 32, 33, 128, 1025])
def test_ray_to_samples_bit_exact(S):
    c = ctx()
    rng = np.random.RandomState(S)
    R = 257 if S < 1025 else 7
    o, d = rng.randn(R, 3).astype(F32), rng.randn(R, 3).astype(F32)
    near = rng.uniform(0.1, 1, R).astype(F32)
    far = (near + rng.uniform(0.5, 5, R)).astype(F32)
    tr = rng.rand(R, S).astype(F32)
    tr[0, :] = 0.0
    tr[1, :] = 1.0
    od, dd, nd, fd, trd = cu(o), cu(d), cu(near), cu(far), cu(tr)      # held: the launches read them asynchronously
    for lindisp in (0, 1):
        for per_ray in (True, False):
            for t_rand in (None, tr):
                pts, dirs, z = (torch.empty(R, S, 3, device=DEV), torch.empty(R, S, 3, device=DEV), torch.empty(R, S, device=DEV))
                nv, fv = (nd, fd) if per_ray else (None, None)
                c.check(c.lib.nm_ray_to_samples(c.h, _p(od), _p(dd), _p(nv), _p(fv), 0.25, 3.5, R, S, lindisp,
                                                _p(None if t_rand is None else trd), _p(pts), _p(dirs), _p(z), c.stream()))
                rp, rz = sx.ray_to_samples(o, d, near if per_ray else 0.25, far if per_ray else 3.5, S, bool(lindisp), t_rand)
                tag = f"S={S} lindisp={lindisp} per_ray={per_ray} t_rand={t_rand is not None}"
                exact("z " + tag, z, rz)
                exact("pts " + tag, pts, rp)
                assert torch.equal(dirs, dd[:, None, :].expand(R, S, 3))
    z2 = torch.empty(R, S, device=DEV)                        # z only: pts and dirs NULL, no origins / directions
    c.check(c.lib.nm_ray_to_samples(c.h, None, None, _p(nd), _p(fd), 0.0, 0.0, R, S, 0, None, None, None, _p(z2), c.stream()))
    exact("z only", z2, sx.ray_to_samples(o, d, near, far, S)[1])


def _pdf_rows(R, B, rng):
    w = (rng.rand(R, B - 1) ** 6).astype(F32)
    w[::5] = 0                                                  # all-zero rows: uniform pdf
    w[1::5] = 0
    w[1::5, rng.randint(0, B - 1)] = 3.0                        # single-spike rows
    return w


@pytest.mark.parametrize("B,N", [(17, 11), (64, 100), (200, 33), (1536, 47)])
def test_sample_pdf_bit_exact(B, N):
    c = ctx()
    rng = np.random.RandomState(B)
    R = 41
    bins = np.sort(rng.rand(R, B).astype(F32) * 4, 1)
    w = _pdf_rows(R, B, rng)
    cdf = sx.build_cdf(w)
    u = rng.rand(R, N).astype(F32)
    u[:, 0] = 0.0
    u[:, 1] = cdf[:, -1]                                        # u >= cdf[-1]
    u[:, 2] = 1.0
    k = min(N - 3, B)
    u[:, 3:3 + k] = cdf[:, :k]                                 # u exactly on cdf entries
    for uu in (u, None):
        out = nb.sample_pdf(cu(bins), cu(w), N, det=True, u=None if uu is None else cu(uu))
        exact(f"sample_pdf B={B} N={N} u={'given' if uu is not None else 'linspace'}", out, sx.sample_pdf(bins, w, N, u=uu))
    out = torch.empty(1, 4, device=DEV)
    big = torch.zeros(1, 1537, device=DEV)
    rc = c.lib.nm_sample_pdf(c.h, _p(big), _p(big), 1, 1537, 4, None, _p(out), c.stream())
    assert rc != 0 and b"too many bins" in c.lib.nm_last_error(c.h)


@pytest.mark.parametrize("S,N", [(64, 0), (33, 31), (64, 64), (64, 128), (100, 156), (128, 384), (512, 512),
                                 (1000, 1048), (3, 7), (48, 40)])
def test_importance_bit_exact(S, N):
    """S + N crosses every pow2 from 64 to 2048 (1000 + 1048: 4 x (2 x 999 + 2 x 2048) x 4 B = 95 KB, the opt-in path)."""
    N = N or 33
    rng = np.random.RandomState(S + N)
    R = 45
    o, d = rng.randn(R, 3).astype(F32), rng.randn(R, 3).astype(F32)
    z = np.sort(rng.uniform(0.5, 4, (R, S)).astype(F32), 1)
    w = (rng.rand(R, S) ** 6).astype(F32)
    w[::4] = 0
    w[1::4] = 0
    w[1::4, S // 2] = 1.0
    for inc in (True, False):
        pts, _, zo = nb.ray_to_importance_samples({"origin": cu(o), "direction": cu(d)}, cu(z), cu(w), N, including_old=inc)
        rp, rz = sx.importance(o, d, z, w, N, including_old=inc)
        exact(f"importance z S={S} N={N} old={inc}", zo, rz)
        exact(f"importance pts S={S} N={N} old={inc}", pts, rp)


def test_importance_bitonic_fallback_matches_rank_merge():
    """A 1-ulp inversion in the old z list sends the kernel to its bitonic sort; the sorted union is the same values."""
    rng = np.random.RandomState(9)
    R, S, N = 16, 64, 64
    z = np.sort(rng.uniform(0.5, 4, (R, S)).astype(F32), 1)
    w = (rng.rand(R, S) ** 4).astype(F32)
    zi = z.copy()
    zi[:, 10] = np.nextafter(zi[:, 11], F32(0))
    zi[:, 11] = np.nextafter(zi[:, 11], F32(9))
    zi[:, [10, 11]] = zi[:, [11, 10]]                          # 1-ulp inversion
    o, d = rng.randn(R, 3).astype(F32), rng.randn(R, 3).astype(F32)
    _, _, zb = nb.ray_to_importance_samples({"origin": cu(o), "direction": cu(d)}, cu(zi), cu(w), N)
    exact("bitonic path", zb, sx.importance(o, d, zi, w, N)[1])
    assert (zb[:, 1:] >= zb[:, :-1]).all()
    c = ctx()
    big = torch.zeros(1, 6000, device=DEV)
    out = torch.empty(1, 7000, device=DEV)
    rc = c.lib.nm_importance_samples(c.h, None, None, _p(big), _p(big), 1, 6000, 1000, 1, None, None, _p(out), c.stream())
    assert rc != 0 and b"too many samples" in c.lib.nm_last_error(c.h)


@pytest.mark.parametrize("n_verts", [None, 17, 65])
def test_near_far_bit_exact(n_verts):
    """nm_near_far (k_near_far) and the frame path nm_near_far_mesh (k_near_far_groups) against the exhaustive loop, on
    rays tangent to the outermost vertex spheres and to group cull spheres, from 1, 10 and 50 body radii."""
    V, o, d, thr = near_far_cases(n_verts=n_verts)
    rn, rf = sx.near_far_exhaustive(o, d, V, thr)
    n, f = nb.geometry_guided_near_far(cu(o), cu(d), cu(V), thr)
    exact("near_far near", n, rn)
    exact("near_far far", f, rf)
    faces = np.zeros((1, 3), np.int32)
    actor = 3
    ops.set_mesh(V, faces, None, actor=actor)                   # host vertices: builds the vertex groups
    n, f = ops.near_far_mesh(cu(o), cu(d), actor, thr)
    exact("near_far_mesh near", n, rn)
    exact("near_far_mesh far", f, rf)


@pytest.mark.parametrize("S", [1, 2, 31, 32, 33, 384, 640, 1024])
def test_composite_forward_windows(S):
    R = 48 if S <= 640 else 12
    raw, z, d = _composite_inputs(S, R, S)
    raw[-3:, :, 3] = -5.0                                       # all-transparent rays
    raw[-6:-3, 0, 3] = 1e4                                      # opaque from the first sample
    noise = np.random.RandomState(S + 1).randn(R, S).astype(F32) * 0.5
    for scale, nz in ((1.0, None), (0.37, noise)):
        for wb in (True, False):
            got = nb.raw2outputs(cu(raw), cu(z), cu(d), raw_noise_std=0.5 if nz is not None else 0, noise=None if nz is None else cu(nz),
                                 white_bkg=wb, sigma_scale=scale)
            win = sx.composite_forward(raw, z, d, noise=nz, sigma_scale=scale, white_bkg=wb)
            for name, t in zip(("rgb", "disp", "acc", "w", "depth"), got):
                msg = sx.outside(f"{name} S={S} scale={scale} white={wb}", t.cpu().numpy(), win[name])
                assert msg is None, msg


def _backward(raw, z, d, grads, noise=None, scale=1.0, wb=True):
    c = ctx()
    R, S = z.shape
    g = [None if x is None else cu(x) for x in grads]
    rd, zd, dd, nz = cu(raw), cu(z), cu(d), None if noise is None else cu(noise)     # held until the result is read
    out = torch.empty(R, S, 4, device=DEV)
    c.check(c.lib.nm_raw2outputs_backward(c.h, _p(rd), _p(zd), _p(dd), R, S, _p(nz), float(scale), int(wb), _p(g[0]), _p(g[1]),
                                          _p(g[2]), _p(g[3]), _p(out), c.stream()))
    return out.cpu().numpy()


@pytest.mark.parametrize("S", [1, 2, 31, 32, 33, 384, 640, 1024])
def test_composite_backward_windows(S):
    """d raw of every element inside its own window, on rays with an opaque surface (sigma * delta from 5 to 40) and
    random gradients; every combination of NULL gradient inputs is its own window, and the sum of the single ones."""
    R = 48 if S <= 640 else 12
    raw, z, d = _composite_inputs(S + 100, R, S)
    rng = np.random.RandomState(S)
    noise = rng.randn(R, S).astype(F32) * 0.5
    grads = [rng.randn(R, 3).astype(F32), rng.randn(R).astype(F32), rng.randn(R).astype(F32), rng.randn(R, S).astype(F32)]
    for scale, nz, wb in ((1.0, None, True), (0.37, noise, False)):
        got = _backward(raw, z, d, grads, nz, scale, wb)
        win = sx.composite_backward(raw, z, d, *grads, noise=nz, sigma_scale=scale, white_bkg=wb)
        msg = sx.outside(f"d raw S={S} scale={scale} white={wb}", got, win)
        assert msg is None, msg
    single = []
    for mask in range(1, 16):
        gs = [g if mask >> k & 1 else None for k, g in enumerate(grads)]
        got = _backward(raw, z, d, gs)
        win = sx.composite_backward(raw, z, d, *gs)
        msg = sx.outside(f"d raw with gradients {mask:04b}", got, win)
        assert msg is None, msg
        if mask in (1, 2, 4, 8):
            single.append((got, win))
        if mask == 15:
            total = sum(s[0].astype(np.float64) for s in single)
            B = win.B + sum(s[1].B for s in single)
            assert (np.abs(got - total) <= B).all()


def test_composite_backward_opaque_surface():
    """The case that separates an exclusive suffix summed directly from one formed as inclusive - own term: one ray, 64
    samples on z in [2, 6], one surface sample of sigma 50 / 150 / 300."""
    rng = np.random.RandomState(0)
    R, S = 12, 64
    z = np.sort(rng.uniform(2, 6, (R, S)), 1).astype(F32)
    raw = rng.randn(R, S, 4).astype(F32)
    raw[:, 20, 3] = np.repeat([50.0, 150.0, 300.0], 4)
    d = np.tile(np.array([[0, 0, 1]], F32), (R, 1))
    g = rng.randn(R, 3).astype(F32)
    got = _backward(raw, z, d, [g, None, None, None])
    win = sx.composite_backward(raw, z, d, g_rgb=g)
    rel = np.abs(got[:, 20, 3] - win.e[:, 20, 3]) / np.abs(win.e[:, 20, 3])
    print("relative error of the surface sample's sigma gradient:", rel, "window:", win.B[:, 20, 3] / np.abs(win.e[:, 20, 3]))
    msg = sx.outside("d raw", got, win)
    assert msg is None, msg


@pytest.mark.parametrize("sizes", [(32,), (1, 32), (33,), (5, 7, 9, 11, 1, 100, 200, 300, 392), (1025,),
                                   (4096,), (512,) * 8, (4000, 96), (3,) * 9])
def test_merge_bit_exact(sizes):
    c = ctx()
    rng = np.random.RandomState(len(sizes) + sum(sizes))
    R = 13
    zs = [np.round(rng.rand(R, s) * 64).astype(F32) / 16 for s in sizes]      # exact ties across lists, unsorted
    raws = [rng.randn(R, s, 4).astype(F32) for s in sizes]
    zt, rt = ops.merge_samples([cu(z) for z in zs], [cu(r) for r in raws])
    want_z, want_r = sx.merge(zs, raws)
    exact(f"merge z {sizes}", zt, want_z)
    exact(f"merge raw {sizes}", rt, want_r)
    n = len(sizes)
    zl = [cu(z) for z in zs]
    zo = torch.empty(R, sum(sizes), device=DEV)
    c.check(c.lib.nm_merge_samples(c.h, n, (C.c_void_p * n)(*[z.data_ptr() for z in zl]), None, (C.c_int32 * n)(*sizes), R,
                                   _p(zo), None, c.stream()))
    exact("merge z without raw", zo, want_z)


def test_merge_limits():
    c = ctx()
    z = [torch.zeros(2, 4000, device=DEV), torch.zeros(2, 97, device=DEV)]
    zo = torch.empty(2, 4097, device=DEV)
    rc = c.lib.nm_merge_samples(c.h, 2, (C.c_void_p * 2)(*[t.data_ptr() for t in z]), None, (C.c_int32 * 2)(4000, 97), 2,
                                _p(zo), None, c.stream())
    assert rc != 0 and b"more than 4096" in c.lib.nm_last_error(c.h)
    ten = [torch.zeros(2, 3, device=DEV)] * 10
    rc = c.lib.nm_merge_samples(c.h, 10, (C.c_void_p * 10)(*[t.data_ptr() for t in ten]), None, (C.c_int32 * 10)(*[3] * 10), 2,
                                _p(zo), None, c.stream())
    assert rc != 0
