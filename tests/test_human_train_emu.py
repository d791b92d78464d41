"""The human trainer's forward / adjoint kernels (neuman_b200/csrc/human_train_kernels.cuh, smpl_train_kernels.cuh)
executed on the host by the serial emulation in tests/emu/ -- the SAME kernel bodies libneuman_b200.so compiles for
sm_90a -- against torch autograd of the oracle restatement of the reference's lines (utils/ray_utils.py:69-93,
trainers/human_nerf_trainer.py:263-276, models/human_nerf.py:92-122, models/smpl.py:266-505).  This is the CPU half of
the parity check (no GPU in the build container); tests/test_gpu_human_train.py repeats it through the CUDA library."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from oracle import neuman_oracle as no
from oracle import synth_smpl
from tests import emu
from tests.emu import f32, f64, i32, ptr


def _case(seed=3, R=24, S=16):
    body = synth_smpl.random_body(seed=seed, center=(0.0, 0.1, 0.2))
    V = body["verts"].astype(np.float32)
    F = np.ascontiguousarray(np.asarray(body["faces"])[:, :3], dtype=np.int32)
    rng = np.random.RandomState(seed)
    # rays through the body: consecutive samples along a segment, as ray_to_samples makes them
    a = V[rng.randint(0, V.shape[0], R)] + rng.normal(0, 0.05, (R, 3))
    d = rng.normal(0, 1, (R, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    t = np.linspace(-0.12, 0.12, S)
    P = (a[:, None] + t[None, :, None] * d[:, None]).astype(np.float32)
    Sd, I, Cl = mo.signed_distance(P.reshape(-1, 3), V, F)
    T = np.ascontiguousarray(body["Ts"][:V.shape[0]].astype(np.float32).reshape(-1, 16))
    off = rng.normal(0, 0.01, (R, S, 3)).astype(np.float32)
    return V, F, T, P, I.astype(np.int32), Cl, off


def test_warp_diff_forward_and_backward_kernels():
    L = emu.lib()
    V, F, T, P, I, Cl, off = _case()
    R, S, _ = P.shape
    n = R * S
    # ---- forward: T_interp_inv, canonical points (+ offset), directions ----
    Tinv = np.zeros((n, 16), np.float32)
    cp = np.zeros((n, 3), np.float32)
    cd = np.zeros((n, 3), np.float32)
    L.emu_wd_forward(ptr(I), ptr(f64(Cl)), ptr(V), ptr(F), ptr(T), ptr(f32(P)), ptr(off), C.c_longlong(n), ptr(Tinv), ptr(cp))
    L.emu_wd_dirs(ptr(cp), C.c_longlong(R), C.c_int(S), ptr(cd))
    Vt, Tt = torch.from_numpy(V).requires_grad_(True), torch.from_numpy(T).reshape(-1, 4, 4).requires_grad_(True)
    offt = torch.from_numpy(off).requires_grad_(True)
    Ti_o = no.warp_diff_Tinv(Cl, I, Vt, F, Tt)
    cp_o, cd_o = no.eval_human_samples(torch.from_numpy(P), Cl, I, Vt, F, Tt, offt)
    assert np.abs(Tinv.reshape(-1, 4, 4) - Ti_o.detach().numpy()).max() < 2e-6 * max(1.0, float(Ti_o.detach().abs().max()))
    assert np.abs(cp.reshape(R, S, 3) - cp_o.detach().numpy()).max() < 2e-6
    assert np.abs(cd.reshape(R, S, 3) - cd_o.detach().numpy()).max() < 2e-5
    # ---- backward, drop-in form: gradient of T_interp_inv -> T, verts ----
    rng = np.random.RandomState(1)
    gTi = rng.normal(0, 1, (n, 16)).astype(np.float32)
    (Ti_o * torch.from_numpy(gTi).reshape(n, 4, 4)).sum().backward()
    gT, gV = np.zeros_like(T), np.zeros_like(V)
    L.emu_wd_backward(ptr(I), ptr(f64(Cl)), ptr(V), ptr(F), ptr(T), None, ptr(gTi), None, C.c_longlong(n), ptr(gT), ptr(gV))
    wT, wV = Tt.grad.numpy().reshape(-1, 16), Vt.grad.numpy()
    assert np.abs(gT - wT).max() < 2e-4 * (1 + np.abs(wT).max()), (np.abs(gT - wT).max(), np.abs(wT).max())
    assert np.abs(gV - wV).max() < 2e-4 * (1 + np.abs(wV).max()), (np.abs(gV - wV).max(), np.abs(wV).max())
    # ---- backward, fused form: gradients of (can_pts, can_dirs) -> T, verts, offset ----
    Vt.grad = Tt.grad = None
    g_cp = rng.normal(0, 1, (R, S, 3)).astype(np.float32)
    g_cd = rng.normal(0, 1, (R, S, 3)).astype(np.float32)
    ((cp_o * torch.from_numpy(g_cp)).sum() + (cd_o * torch.from_numpy(g_cd)).sum()).backward()
    g_tot = np.zeros((n, 3), np.float32)
    L.emu_wd_dirs_backward(ptr(cp), ptr(g_cp), ptr(g_cd), C.c_longlong(R), C.c_int(S), ptr(g_tot))
    w_off = offt.grad.numpy().reshape(-1, 3)
    assert np.abs(g_tot - w_off).max() < 2e-4 * (1 + np.abs(w_off).max())
    gT[:], gV[:] = 0, 0
    L.emu_wd_backward(ptr(I), ptr(f64(Cl)), ptr(V), ptr(F), ptr(T), ptr(f32(P)), None, ptr(g_tot), C.c_longlong(n), ptr(gT), ptr(gV))
    wT, wV = Tt.grad.numpy().reshape(-1, 16), Vt.grad.numpy()
    assert np.abs(gT - wT).max() < 2e-4 * (1 + np.abs(wT).max()), (np.abs(gT - wT).max(), np.abs(wT).max())
    assert np.abs(gV - wV).max() < 2e-4 * (1 + np.abs(wV).max()), (np.abs(gV - wV).max(), np.abs(wV).max())
    # each of the two gradient inputs alone (null pointers on the other)
    only = np.zeros((n, 3), np.float32)
    L.emu_wd_dirs_backward(ptr(cp), None, ptr(g_cd), C.c_longlong(R), C.c_int(S), ptr(only))
    assert np.abs((only + g_cp.reshape(-1, 3)) - g_tot).max() < 1e-5


@pytest.mark.parametrize("zero_joints", [False, True])
def test_smpl_scene_forward_and_backward_kernels(zero_joints):
    """HumanNeRF.vertex_forward (models/human_nerf.py:92-122) and its adjoint to poses / betas / alignments; also with joints
    whose axis-angle is exactly zero (the Rodrigues formula of models/smpl.py:422 divides by |r + 1e-8|)."""
    L = emu.lib()
    model = synth_smpl.torch_model(0)
    nv, nj, nb = model["v_template"].shape[0], model["parents"].shape[0], model["shapedirs"].shape[-1]
    rng = np.random.RandomState(4)
    p0 = rng.normal(0, 0.3, (1, 3 * nj))
    if zero_joints:
        p0[0, 0:3] = 0.0
        p0[0, 15:27] = 0.0
    pose = torch.from_numpy(p0).float().requires_grad_(True)
    betas = torch.from_numpy(rng.normal(0, 1.0, (1, nb))).float().requires_grad_(True)
    ang = 0.2
    align = np.eye(4, dtype=np.float32)
    align[:3, :3] = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]])
    align = align.T.copy()
    align[3, :3] = (0.3, -0.1, 2.0)
    align = torch.from_numpy(align).requires_grad_(True)
    scale = 0.4
    world_o, T_o = no.vertex_forward(model, pose, betas, align, scale)
    # LBS intermediates from the (reference-validated) oracle; on the GPU they come from the forward LBS kernels
    with torch.no_grad():
        da = no.da_pose(nj)
        T_pose, v_shaped = no.smpl_lbs(model, pose, betas)
        T_da, _ = no.smpl_lbs(model, da, betas)
        J = torch.einsum("ik,ji->jk", v_shaped, model["J_regressor"])
    Tp, Td = f32(T_pose.numpy().reshape(-1, 16)), f32(T_da.numpy().reshape(-1, 16))
    rest, Jn = f32(v_shaped.numpy()), f32(J.numpy())
    al = f32(align.detach().numpy())
    T_out, world = np.zeros((nv, 16), np.float32), np.zeros((nv, 3), np.float32)
    L.emu_smplt_scene_forward(ptr(Tp), ptr(Td), ptr(rest), ptr(al), C.c_float(scale), C.c_int(nv), ptr(T_out), ptr(world))
    assert np.abs(T_out.reshape(-1, 4, 4) - T_o[0].detach().numpy()).max() < 5e-6
    assert np.abs(world - world_o[0].detach().numpy()).max() < 5e-6
    # ---- backward ----
    gT = rng.normal(0, 1, (nv, 16)).astype(np.float32)
    gw = rng.normal(0, 1, (nv, 3)).astype(np.float32)
    ((T_o[0] * torch.from_numpy(gT).reshape(nv, 4, 4)).sum() + (world_o[0] * torch.from_numpy(gw)).sum()).backward()
    W, Jreg = f32(model["weights"].numpy()), f32(model["J_regressor"].numpy())
    sd = f32(model["shapedirs"].numpy().reshape(nv * 3, nb))
    par = i32(model["parents"].numpy())
    z = lambda *s: np.zeros(s, np.float32)
    gP, gD, grest, gpre, gAp, gAd, gJ = z(nv, 16), z(nv, 16), z(nv, 3), z(16), z(nj, 16), z(nj, 16), z(nj, 3)
    g_pose, g_betas, g_align = z(nj * 3), z(nb), z(16)
    L.emu_smplt_scene_backward(ptr(Tp), ptr(Td), ptr(rest), ptr(Jn), ptr(f32(pose.detach().numpy())), ptr(f32(da.numpy())),
                               ptr(al), C.c_float(scale), ptr(W), ptr(Jreg), ptr(sd), ptr(par), C.c_int(nv), C.c_int(nj),
                               C.c_int(nb), ptr(gT), ptr(gw), ptr(gP), ptr(gD), ptr(grest), ptr(gpre), ptr(gAp), ptr(gAd),
                               ptr(gJ), ptr(g_pose), ptr(g_betas), ptr(g_align))
    for name, got, want in (("pose", g_pose, pose.grad.numpy().reshape(-1)), ("betas", g_betas, betas.grad.numpy().reshape(-1)),
                            ("alignment", g_align, align.grad.numpy().reshape(-1))):
        err, ref = np.abs(got - want).max(), np.abs(want).max()
        assert err < 5e-4 * (1 + ref), (name, err, ref)


# ---------------------------------------------------------------------------------------------
# The Python binding layer (neuman_b200/autograd.py: argument order, shapes, which gradients are returned) dry-run on
# CPU tensors: a stand-in library object routes the nm_* calls of the human-trainer entry points to the emulated kernels
# (the LBS forward intermediates, which libneuman_b200.so computes with its shared-memory kernels, come from the oracle).
# ---------------------------------------------------------------------------------------------
def _arr(p, n, ctype=C.c_float):
    return np.ctypeslib.as_array((ctype * n).from_address(p.value))


class _EmuLib:
    def __init__(self, model):
        self.L, self.model = emu.lib(), model

    def nm_warp_diff_forward(self, h, f_id, closest, v, faces, t, n, Tinv, st):
        self.L.emu_wd_forward(f_id, closest, v, faces, t, None, None, C.c_longlong(n), Tinv, None)
        return 0

    def nm_warp_diff_backward(self, h, f_id, closest, v, faces, t, n, g, nv, g_T, g_v, st):
        for p, k in ((g_T, 16), (g_v, 3)):
            if p.value:
                C.memset(p, 0, nv * k * 4)
        self.L.emu_wd_backward(f_id, closest, v, faces, t, None, g, None, C.c_longlong(n), g_T, g_v)
        return 0

    def nm_human_canonicalize(self, h, f_id, closest, v, faces, t, p, off, R, S, cp, cd, st):
        self.L.emu_wd_forward(f_id, closest, v, faces, t, p, off, C.c_longlong(R * S), None, cp)
        self.L.emu_wd_dirs(cp, C.c_longlong(R), C.c_int(S), cd)
        return 0

    def nm_human_canonicalize_backward(self, h, f_id, closest, v, faces, t, p, cp, g_cp, g_cd, R, S, nv, g_off, g_T, g_v, st):
        for q, k in ((g_T, 16), (g_v, 3)):
            if q.value:
                C.memset(q, 0, nv * k * 4)
        self.L.emu_wd_dirs_backward(cp, g_cp, g_cd, C.c_longlong(R), C.c_int(S), g_off)
        self.L.emu_wd_backward(f_id, closest, v, faces, t, p, None, g_off, C.c_longlong(R * S), g_T, g_v)
        return 0

    def _lbs(self, pose, da, betas):
        m = self.model
        with torch.no_grad():
            pt, bt = torch.from_numpy(pose.copy())[None], torch.from_numpy(betas.copy())[None]
            T_pose, v_shaped = no.smpl_lbs(m, pt, bt)
            T_da, _ = no.smpl_lbs(m, torch.from_numpy(da.copy())[None], bt)
            J = torch.einsum("ik,ji->jk", v_shaped, m["J_regressor"])
        return (f32(T_pose.numpy().reshape(-1, 16)), f32(T_da.numpy().reshape(-1, 16)), f32(v_shaped.numpy()), f32(J.numpy()))

    def nm_smpl_scene_forward_train(self, h, model, p, da, b, a, scale, T, world, st):
        nj, nb = self.model["parents"].shape[0], self.model["shapedirs"].shape[-1]
        Tp, Td, rest, J = self._lbs(_arr(p, 3 * nj), _arr(da, 3 * nj), _arr(b, nb))
        self.L.emu_smplt_scene_forward(ptr(Tp), ptr(Td), ptr(rest), a, C.c_float(scale), C.c_int(rest.shape[0]), T, world)
        return 0

    def nm_smpl_scene_backward(self, h, model, p, da, b, a, scale, g_T, g_world, g_pose, g_betas, g_align, st):
        m = self.model
        nv, nj, nb = m["v_template"].shape[0], m["parents"].shape[0], m["shapedirs"].shape[-1]
        pose, dap = _arr(p, 3 * nj), _arr(da, 3 * nj)
        Tp, Td, rest, J = self._lbs(pose, dap, _arr(b, nb))
        z = lambda *s: np.zeros(s, np.float32)
        keep = [z(nv, 16), z(nv, 16), z(nv, 3), z(16), z(nj, 16), z(nj, 16), z(nj, 3)]
        W, Jreg = f32(m["weights"].numpy()), f32(m["J_regressor"].numpy())
        sd, par = f32(m["shapedirs"].numpy().reshape(nv * 3, nb)), i32(m["parents"].numpy())
        self.L.emu_smplt_scene_backward(ptr(Tp), ptr(Td), ptr(rest), ptr(J), p, da, a, C.c_float(scale), ptr(W), ptr(Jreg), ptr(sd),
                                        ptr(par), C.c_int(nv), C.c_int(nj), C.c_int(nb), g_T, g_world, *[ptr(k) for k in keep],
                                        g_pose, g_betas, g_align)
        return 0


class _EmuCtx:
    h = None

    def __init__(self, model):
        self.lib = _EmuLib(model)

    def check(self, rc):
        assert rc == 0

    def stream(self):
        return None


def test_autograd_bindings_on_the_emulated_library(monkeypatch):
    import contextlib
    from neuman_b200 import autograd as nag, ops
    model = synth_smpl.torch_model(0)
    ctx = _EmuCtx(model)
    monkeypatch.setattr(nag, "_ctx_for", lambda t: ctx)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    V, F, T, P, I, Cl, off = _case(seed=5, R=12, S=9)
    R, S, _ = P.shape
    f_id, closest = torch.from_numpy(I), torch.from_numpy(f64(Cl))
    verts, Tt = torch.from_numpy(V).requires_grad_(True), torch.from_numpy(T.reshape(-1, 4, 4).copy()).requires_grad_(True)
    offt = torch.from_numpy(off).requires_grad_(True)
    Vo, To, offo = (x.detach().clone().requires_grad_(True) for x in (verts, Tt, offt))
    rng = np.random.RandomState(2)
    # T_interp_inv
    Ti = nag.warp_diff_tinv(verts, Tt, f_id, closest, F)
    Ti_o = no.warp_diff_Tinv(Cl, I, Vo, F, To)
    w = torch.from_numpy(rng.normal(0, 1, (R * S, 4, 4)).astype(np.float32))
    (Ti * w).sum().backward()
    (Ti_o * w).sum().backward()
    assert Tt.grad.shape == (V.shape[0], 4, 4)
    assert (Tt.grad - To.grad).abs().max() < 2e-4 * (1 + To.grad.abs().max())
    assert (verts.grad - Vo.grad).abs().max() < 2e-4 * (1 + Vo.grad.abs().max())
    # fused, with and without an offset / with only some inputs requiring grad
    verts.grad = Tt.grad = Vo.grad = To.grad = None
    cp, cd = nag.human_canonicalize(torch.from_numpy(P), verts, Tt, f_id, closest, F, offt)
    cp_o, cd_o = no.eval_human_samples(torch.from_numpy(P), Cl, I, Vo, F, To, offo)
    w1, w2 = (torch.from_numpy(rng.normal(0, 1, (R, S, 3)).astype(np.float32)) for _ in range(2))
    ((cp * w1).sum() + (cd * w2).sum()).backward()
    ((cp_o * w1).sum() + (cd_o * w2).sum()).backward()
    for got, want in ((offt.grad, offo.grad), (Tt.grad, To.grad), (verts.grad, Vo.grad)):
        assert got.shape == want.shape and (got - want).abs().max() < 2e-4 * (1 + want.abs().max())
    cp2, cd2 = nag.human_canonicalize(torch.from_numpy(P), verts.detach(), Tt.detach().requires_grad_(True), f_id, closest, F, None)
    assert (cp2 - (cp_o - offo).detach()).abs().max() < 2e-6
    cd2.sum().backward()
    # vertex_forward
    nj, nb = model["parents"].shape[0], model["shapedirs"].shape[-1]
    dm = ops.SmplModelDevice(model["v_template"], model["shapedirs"], model["J_regressor"], model["weights"], model["parents"],
                             device="cpu")
    pose = torch.from_numpy(rng.normal(0, 0.3, (1, 3 * nj)).astype(np.float32)).requires_grad_(True)
    betas = torch.from_numpy(rng.normal(0, 1.0, (1, nb)).astype(np.float32)).requires_grad_(True)
    al = torch.eye(4)
    al[3, :3] = torch.tensor([0.3, -0.1, 2.0])
    al.requires_grad_(True)
    po, bo, ao = (x.detach().clone().requires_grad_(True) for x in (pose, betas, al))
    world, Tw = nag.vertex_forward(dm, pose, betas, al, 0.4, no.da_pose(nj))
    world_o, T_o = no.vertex_forward(model, po, bo, ao, 0.4)
    assert world.shape == world_o.shape and Tw.shape == T_o.shape
    assert (Tw - T_o).abs().max() < 5e-6 and (world - world_o).abs().max() < 5e-6
    g1, g2 = torch.from_numpy(rng.normal(0, 1, tuple(Tw.shape)).astype(np.float32)), torch.from_numpy(rng.normal(0, 1, tuple(world.shape)).astype(np.float32))
    ((Tw * g1).sum() + (world * g2).sum()).backward()
    ((T_o * g1).sum() + (world_o * g2).sum()).backward()
    for got, want in ((pose.grad, po.grad), (betas.grad, bo.grad), (al.grad, ao.grad)):
        assert got.shape == want.shape and (got - want).abs().max() < 5e-4 * (1 + want.abs().max())


@pytest.mark.parametrize("R,S", [(1, 2), (3, 2), (5, 7), (1, 33)])
def test_warp_diff_kernels_edge_shapes(R, S):
    """Smallest legal ray (two samples: the second direction is the copy of the first), single rays, sizes that do not fill
    a block; optional outputs left out (null pointers)."""
    L = emu.lib()
    V, F, T, P, I, Cl, off = _case(seed=11, R=R, S=S)
    n = R * S
    cp, cd = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.float32)
    L.emu_wd_forward(ptr(I), ptr(f64(Cl)), ptr(V), ptr(F), ptr(T), ptr(f32(P)), None, C.c_longlong(n), None, ptr(cp))
    L.emu_wd_dirs(ptr(cp), C.c_longlong(R), C.c_int(S), ptr(cd))
    Vt, Tt = torch.from_numpy(V).requires_grad_(True), torch.from_numpy(T).reshape(-1, 4, 4).requires_grad_(True)
    cp_o, cd_o = no.eval_human_samples(torch.from_numpy(P), Cl, I, Vt, F, Tt, None)
    assert np.abs(cp.reshape(R, S, 3) - cp_o.detach().numpy()).max() < 2e-6
    assert np.abs(cd.reshape(R, S, 3) - cd_o.detach().numpy()).max() < 5e-5
    assert np.abs(cd.reshape(R, S, 3)[:, -1] - cd.reshape(R, S, 3)[:, -2]).max() == 0          # last direction = the previous one
    rng = np.random.RandomState(R * 100 + S)
    g_cd = rng.normal(0, 1, (R, S, 3)).astype(np.float32)
    (cd_o * torch.from_numpy(g_cd)).sum().backward()
    g_tot = np.zeros((n, 3), np.float32)
    L.emu_wd_dirs_backward(ptr(cp), None, ptr(g_cd), C.c_longlong(R), C.c_int(S), ptr(g_tot))
    gT = np.zeros_like(T)
    L.emu_wd_backward(ptr(I), ptr(f64(Cl)), ptr(V), ptr(F), ptr(T), ptr(f32(P)), None, ptr(g_tot), C.c_longlong(n), ptr(gT), None)   # no vertex gradient wanted
    wT = Tt.grad.numpy().reshape(-1, 16)
    assert np.abs(gT - wT).max() < 5e-4 * (1 + np.abs(wT).max())
    gV = np.zeros_like(V)
    L.emu_wd_backward(ptr(I), ptr(f64(Cl)), ptr(V), ptr(F), ptr(T), ptr(f32(P)), None, ptr(g_tot), C.c_longlong(n), None, ptr(gV))   # only the vertex gradient
    wV = Vt.grad.numpy()
    assert np.abs(gV - wV).max() < 5e-4 * (1 + np.abs(wV).max())
