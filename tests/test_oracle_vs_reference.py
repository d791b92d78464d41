"""The oracle restatement (oracle/neuman_oracle.py) against what the UNMODIFIED reference returned on the same inputs
(tests/golden/reference.npz, written by tools/make_golden_reference.py).  Runs anywhere (no GPU, no reference tree).
Networks are rebuilt with neuman_b200's mirror under the reference's seed; their parameter checksums must equal the
reference's, so the comparisons are made on the very weights the reference used."""
import os
import tempfile

import numpy as np
import pytest
import torch

import neuman_b200 as nb
from oracle import neuman_oracle as no
from oracle import synth_smpl

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference.npz")


@pytest.fixture(autouse=True, scope="module")
def _one_thread():
    """CPU float32 reductions round differently with the number of threads they are split over; the stored outputs were
    computed on one thread, so the comparisons run on one thread too (the same results on any host)"""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


@pytest.fixture(scope="module")
def g():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


# ---- inputs (shared with tools/make_golden_reference.py) ----
def _camera(H, W, f=None, seed=0):
    rng = np.random.RandomState(seed)
    f = f or 1000.0 * W / 1280
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1.0]])
    a = rng.uniform(-0.2, 0.2)
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    c2w = np.eye(4)
    c2w[:3, :3] = R
    c2w[:3, 3] = [0.1, -0.05, -1.5]
    return K, c2w


def _sampling_inputs():
    torch.manual_seed(0)
    R, S, N = 37, 24, 16
    o, d = torch.randn(R, 3), torch.nn.functional.normalize(torch.randn(R, 3), dim=-1)
    near, far = torch.rand(R, 1), 2 + torch.rand(R, 1)
    raw = torch.randn(R, S, 4) * 3
    return o, d, near, far, raw, S, N


def _net_inputs():
    torch.manual_seed(2)
    return torch.randn(50, 7, 3), torch.nn.functional.normalize(torch.randn(50, 7, 3), dim=-1)


def _rows(n):
    """the fixed sample of vertex / transform rows stored for the per-vertex SMPL outputs (files stay small): 512 seeded
    rows plus the last 24 (the joints, where they are appended)"""
    return np.unique(np.concatenate([np.random.RandomState(7).choice(n, 512, replace=False), np.arange(n - 24, n)]))


def _checksum(module):
    """sum and sum of squares of every parameter and buffer, in float64"""
    t = [p.detach().double() for p in module.state_dict().values()]
    return np.array([sum(float(x.sum()) for x in t), sum(float((x * x).sum()) for x in t)])


def _grad_summary(t):
    """a gradient as sum, sum of |x|, sum of squares (float64) and its first 64 values"""
    x = t.detach().double().reshape(-1)
    head = np.zeros(64)
    head[:min(64, x.numel())] = x[:64].numpy()
    return np.concatenate([[float(x.sum()), float(x.abs().sum()), float((x * x).sum())], head])


def _near_far_inputs():
    rng = np.random.RandomState(0)
    V = rng.normal(0, 0.3, size=(500, 3)).astype(np.float32)
    o = np.tile(np.array([[0, 0, -2.0]], dtype=np.float32), (64, 1))
    d = rng.normal(0, 0.3, size=(64, 3)).astype(np.float32) + np.array([0, 0, 1], dtype=np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return o, d, V


def _smpl_inputs():
    rng = np.random.RandomState(3)
    return torch.from_numpy(rng.normal(0, 0.3, (1, 72))).float(), torch.from_numpy(rng.normal(0, 1, (1, 10))).float()


def _warp_inputs():
    body = synth_smpl.random_body(seed=2)
    rng = np.random.RandomState(0)
    pts = (body["verts"].mean(0) + rng.normal(0, 0.25, size=(6, 9, 3))).astype(np.float32)
    faces6 = np.concatenate([body["faces"], body["faces"]], 1)       # 6-column faces like read_obj
    return pts, body, faces6


def _boost(net):
    with torch.no_grad():      # default init leaves sigma<0 over the whole (small) body region
        net.coarse_human_net.nerf.alpha_linear.weight *= 8
        net.coarse_human_net.nerf.alpha_linear.bias += 0.3


def _human_parts(net):
    """the three networks the human / hybrid renderers evaluate"""
    return torch.nn.ModuleList([net.coarse_human_net, net.coarse_bkg_net, net.fine_bkg_net])


def _human_inputs():
    body = synth_smpl.random_body(seed=1, center=(0.1, 0.0, 0.3))
    body2 = synth_smpl.random_body(seed=4, center=(-0.2, 0.0, 0.5))
    H, W = 10, 8
    K, c2w = _camera(H, W, f=14.0)
    return body, body2, H, W, K, c2w


def _vf_inputs():
    rng = np.random.RandomState(6)
    pose, betas = rng.normal(0, 0.3, (1, 72)).astype(np.float32), rng.normal(0, 1, (1, 10)).astype(np.float32)
    align = np.eye(4, dtype=np.float32)
    align[:3, :3] = np.array([[np.cos(0.2), 0, np.sin(0.2)], [0, 1, 0], [-np.sin(0.2), 0, np.cos(0.2)]])
    align = align.T.copy()
    align[3, :3] = (0.3, -0.1, 2.0)
    return pose, betas, align


def _vertex_cotangents(T_shape, w_shape):
    rng = np.random.RandomState(0)
    g1 = torch.from_numpy(rng.normal(0, 1, tuple(T_shape)).astype(np.float32))
    g2 = torch.from_numpy(rng.normal(0, 1, tuple(w_shape)).astype(np.float32))
    return g1, g2


def _diff_warp_inputs():
    body = synth_smpl.random_body(seed=3)
    V = torch.from_numpy(body["verts"]).float().requires_grad_(True)
    F = np.asarray(body["faces"])[:, :3]
    T = torch.from_numpy(body["Ts"][:6890]).float().requires_grad_(True)
    rng = np.random.RandomState(0)
    P = (body["verts"][rng.randint(0, 6890, 400)] + rng.normal(0, 0.03, (400, 3))).astype(np.float32)
    return P, body, V, F, T


def _nets(seed=1, **over):
    torch.manual_seed(seed)
    return nb.build_nerf(nb.default_opt(use_cuda=False, **over))


def _human_net():
    torch.manual_seed(1)
    net = nb.HumanNeRF(nb.default_opt(use_cuda=False, num_offset_nets=1))
    _boost(net)
    return net


# ---- tests ----
def test_rays_match(g):
    H, W = 12, 20
    K32, c2w32 = g["rays.K"], g["rays.c2w"]
    xy = no.all_pixel_coords(H, W)
    assert np.array_equal(xy, np.argwhere(np.ones((H, W)))[:, ::-1])
    o, d = no.shot_rays(K32, c2w32, xy)
    assert np.array_equal(o, g["rays.o"]) and np.array_equal(d, g["rays.d"])
    o, d = no.shot_all_rays(K32, c2w32, H, W)
    assert np.array_equal(o, g["rays.o_all"]) and np.array_equal(d, g["rays.d_all"])


def test_sampling_composite_match(g):
    o, d, near, far, raw, S, N = _sampling_inputs()
    p, v, z = no.ray_to_samples(o, d, near, far, S)
    assert np.array_equal(p.numpy(), g["samp.p"]) and np.array_equal(v.numpy(), g["samp.v"])
    assert np.array_equal(z.numpy(), g["samp.z"])
    out = no.raw2outputs(raw, z, d, white_bkg=True)
    for i, a in enumerate(out):
        assert np.array_equal(a.numpy(), g[f"samp.out{i}"]), i
    p, v, z2 = no.ray_to_importance_samples(o, d, z, out[3], N)
    assert np.array_equal(z2.numpy(), g["samp.imp_z"]) and np.array_equal(p.numpy(), g["samp.imp_p"])
    # stratified: same draws through the global RNG
    torch.manual_seed(5)
    _, _, zp = no.ray_to_samples(o, d, near, far, S, perturb=1.0)
    assert np.array_equal(zp.numpy(), g["samp.z_perturb"])


def test_nets_match(g):
    torch.manual_seed(1)
    coarse, fine = nb.build_nerf(nb.default_opt(use_cuda=False))
    human, _ = nb.build_nerf(nb.default_opt(use_cuda=False, posenc="rotate"))
    pts, views = _net_inputs()
    for name, net in (("coarse", coarse), ("fine", fine), ("human", human)):
        np.testing.assert_array_equal(_checksum(net), g[f"nets.{name}.checksum"])
        with torch.no_grad():
            y = no.net_forward(no.net_params_from_joiner(net), pts, views)
        assert np.abs(y.numpy() - g[f"nets.{name}"]).max() <= 1e-6, name


def test_near_far_match(g):
    o, d, V = _near_far_inputs()
    n_r, f_r = g["nf.n"], g["nf.f"]
    n, f = no.geometry_guided_near_far(o, d, V, 0.1)
    # the discriminant thr^2-(|ov|^2-z0^2) cancels catastrophically; numpy and torch round it
    # differently (reference noise floor ~4e-6), so the two branches agree to 2e-5, same hit set
    assert np.array_equal(np.isinf(n), np.isinf(n_r))
    hit = ~np.isinf(n)
    assert np.allclose(n[hit], n_r[hit], atol=2e-5) and np.allclose(f[hit], f_r[hit], atol=2e-5)
    n, f = no.geometry_guided_near_far(torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(V), 0.1)
    n_r, f_r = torch.from_numpy(g["nf.n_torch"]), torch.from_numpy(g["nf.f_torch"])
    assert torch.allclose(n, n_r, atol=1e-6) and torch.allclose(f, f_r, atol=1e-6)
    assert torch.equal(torch.isinf(n), torch.isinf(n_r))


def test_smpl_match(g):
    model = synth_smpl.torch_model()
    pose, betas = _smpl_inputs()
    T, v = no.smpl_lbs(model, pose, betas, concat_joints=True)
    assert np.allclose(T.numpy()[_rows(T.shape[0])], g["smpl.T"], atol=1e-6)
    assert np.allclose(v.numpy()[_rows(v.shape[0])], g["smpl.v"], atol=1e-6)
    verts, joints = no.smpl_forward_verts(model, pose, betas)
    assert np.allclose(verts.numpy()[_rows(verts.shape[0])], g["smpl.verts"], atol=1e-5)
    assert np.allclose(joints.numpy().reshape(-1, 3), g["smpl.joints"], atol=1e-5)


def test_warp_match(g):
    pts, body, faces6 = _warp_inputs()
    c, d, cl = no.warp_samples_to_canonical(pts, body["verts"], faces6, body["Ts"])
    assert np.allclose(c, g["warp.c"], atol=1e-12) and np.allclose(d, g["warp.d"], atol=1e-9)
    assert np.allclose(cl, g["warp.cl"])


def test_render_vanilla_match(g):
    coarse, fine = _nets()
    H, W = 6, 9
    rgb, dep = no.render_vanilla(no.net_params_from_joiner(coarse), no.net_params_from_joiner(fine),
                                 g["rv.K"], g["rv.c2w"], H, W, 0.0, 3.14,
                                 rays_per_batch=32, samples_per_ray=16, importance_samples_per_ray=8)
    assert np.allclose(rgb.reshape(H, W, 3), g["rv.rgb"], atol=2e-6)
    assert np.allclose(dep.reshape(H, W), g["rv.depth"], atol=2e-6)


def test_render_human_and_hybrid_match(g):
    net = _human_net()
    np.testing.assert_array_equal(_checksum(_human_parts(net)), g["human.checksum"])
    body, body2, H, W, _, _ = _human_inputs()
    Kc, c2wc = g["human.K"], g["human.c2w"]
    faces = body["faces"]
    hp = no.net_params_from_joiner(net.coarse_human_net)
    cb, fb = no.net_params_from_joiner(net.coarse_bkg_net), no.net_params_from_joiner(net.fine_bkg_net)
    geo = body["geo_threshold"]
    for can in (True, False):
        r_r, d_r, a_r = (g[f"human.smpl{int(can)}.{k}"] for k in ("rgb", "depth", "acc"))
        r, d, a = no.render_smpl_nerf(hp, Kc, c2wc, H, W, body["verts"], faces, body["Ts"], rays_per_batch=32,
                                      samples_per_ray=12, render_can=can, geo_threshold=geo, interval_comp=0.7)
        assert 0 < (a_r > 0).sum() < a_r.size          # the test must see hits and misses
        assert np.allclose(r.reshape(H, W, 3), r_r, atol=2e-6) and np.allclose(d.reshape(H, W), d_r, atol=2e-6)
        assert np.allclose(a.reshape(H, W), a_r, atol=2e-6)
    r, d, a = no.render_hybrid_nerf(cb, fb, hp, Kc, c2wc, H, W, 0.0, 3.14, body["verts"], faces, body["Ts"],
                                    rays_per_batch=32, samples_per_ray=12, importance_samples_per_ray=8,
                                    geo_threshold=geo)
    assert np.allclose(r.reshape(H, W, 3), g["human.hybrid.rgb"], atol=2e-6)
    assert np.allclose(d.reshape(H, W), g["human.hybrid.depth"], atol=2e-6)
    r, d = no.render_hybrid_nerf_multi_persons(cb, fb, [hp, hp], Kc, c2wc, H, W, 0.0, 3.14,
                                               [body["verts"], body2["verts"]], [faces, faces],
                                               [body["Ts"], body2["Ts"]], rays_per_batch=32, samples_per_ray=12,
                                               importance_samples_per_ray=8, geo_threshold=geo)
    assert np.allclose(r.reshape(H, W, 3), g["human.multi.rgb"], atol=2e-6)
    assert np.allclose(d.reshape(H, W), g["human.multi.depth"], atol=2e-6)


def test_mirror_human_nerf_state_dict_matches_the_reference(g):
    """The host mirror (neuman_b200.models) creates the reference's parameters -- names, shapes, default-init values in the
    same order -- including the offset nets, so `hybrid_model_state_dict` checkpoints load unchanged (SURVEY.md §8b)."""
    torch.manual_seed(11)
    m = nb.HumanNeRF(nb.default_opt(use_cuda=False, num_offset_nets=2))
    sm = m.state_dict()
    assert list(sm.keys()) == [str(k) for k in g["sd.keys"]]
    for i, (k, t) in enumerate(sm.items()):
        assert ",".join(str(s) for s in t.shape) == str(g["sd.shapes"][i]), k
        assert float(t.double().sum()) == g["sd.sums"][i], k
        head = t.detach().reshape(-1)[:4].double().numpy()
        assert np.array_equal(head, g["sd.head"][i][:head.size]), k
    assert any(k.startswith("offset_nets.1.nerf.output_linear") for k in sm)


def test_vertex_forward_and_its_gradients_match(g):
    """oracle.vertex_forward (what the SMPL training kernels and their adjoint are checked against) vs the reference's
    HumanNeRF.vertex_forward (models/human_nerf.py:92-122): values and the gradients loss.backward() sends to
    poses / betas / alignments."""
    pose, betas, align = _vf_inputs()
    model = synth_smpl.torch_model(0)
    po, bo = torch.from_numpy(pose).requires_grad_(True), torch.from_numpy(betas).requires_grad_(True)
    ao = torch.from_numpy(align).requires_grad_(True)
    w_o, T_o = no.vertex_forward(model, po, bo, ao, 0.4)
    r = _rows(w_o.shape[1])
    assert np.abs(w_o.detach().numpy()[:, r] - g["vf.w"]).max() < 1e-6
    assert np.abs(T_o.detach().numpy()[:, r] - g["vf.T"]).max() < 1e-6
    g1, g2 = _vertex_cotangents(T_o.shape, w_o.shape)
    ((T_o * g1).sum() + (w_o * g2).sum()).backward()
    for a, b in ((g["vf.g_poses"], po.grad), (g["vf.g_betas"], bo.grad), (g["vf.g_align"], ao.grad)):
        b = b.numpy()
        assert np.abs(a - b).max() < 1e-5 * (1 + np.abs(b).max())


def test_differentiable_warp_matches_and_its_vertex_gradient_depends_on_the_tie_rule(g):
    """oracle.warp_diff_Tinv vs the reference's warp_samples_to_canonical_diff (utils/ray_utils.py:69-93) on the same query
    answers.  Then the property that makes libigl's tie rule matter for TRAINING (DESIGN.md §2): where the closest point
    lies on an edge, both adjacent faces give the same inverse transform, but a different gradient with respect to the
    vertices."""
    from oracle import mesh_oracle as mo
    P, body, V, F, T = _diff_warp_inputs()
    rng = np.random.RandomState(0)
    rng.randint(0, 6890, 400), rng.normal(0, 0.03, (400, 3))             # the draws of the sample points
    S, I, C = mo.signed_distance(P, body["verts"], F)
    assert np.array_equal(g["dw.f_id"], I)
    Ti = no.warp_diff_Tinv(C, I, V, F, T)
    assert np.abs(Ti.detach().numpy() - g["dw.Ti"]).max() == 0
    # the other face of every edge-region sample
    L = mo.barycentric_coordinates_tri(C, *(body["verts"][F[I, k]].astype(np.float64) for k in range(3)))
    edges = {}
    for f, tri in enumerate(F):
        for e in ((tri[0], tri[1]), (tri[1], tri[2]), (tri[2], tri[0])):
            edges.setdefault((min(e), max(e)), []).append(f)
    I2, flipped = I.copy(), 0
    for r in range(len(I)):
        z = np.flatnonzero(np.abs(L[r]) < 1e-9)
        if len(z) == 1:
            tri = F[I[r]]
            e = (tri[(z[0] + 1) % 3], tri[(z[0] + 2) % 3])
            other = [f for f in edges[(min(e), max(e))] if f != I[r]]
            if other:
                I2[r], flipped = other[0], flipped + 1
    assert flipped > 40                                                    # edge regions are common, not a corner case
    Ti2 = no.warp_diff_Tinv(C, I2, V, F, T)
    assert (Ti2 - Ti).abs().max() < 1e-5 * Ti.abs().max()                 # same transform ...
    w = torch.from_numpy(rng.normal(0, 1, tuple(Ti.shape)).astype(np.float32))
    gV1 = torch.autograd.grad((Ti * w).sum(), V, retain_graph=True)[0]
    gV2 = torch.autograd.grad((Ti2 * w).sum(), V)[0]
    assert (gV1 - gV2).abs().max() > 0.05 * gV1.abs().max()               # ... different gradient to the vertices
