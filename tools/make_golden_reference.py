"""Writes tests/golden/reference.npz: what the UNMODIFIED reference (apple/ml-neuman) returns on the inputs of
tests/test_oracle_vs_reference.py, so that those comparisons run anywhere without the reference tree.

    NEUMAN_REFERENCE=/path/to/ml-neuman python tools/make_golden_reference.py

The networks the reference builds are not stored: the tests rebuild them with neuman_b200's mirror under the same seed
(bit-identical default-init weights) and check the parameter checksums stored here.
"""
import contextlib
import io
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import, ref_opts, synth_smpl  # noqa: E402
from tests import test_oracle_vs_reference as T  # noqa: E402
from tests.test_host import offset_net_input as H_inputs_offset, module_interface_inputs as H_inputs_module  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference.npz")


def _quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def _cap(ref, K, c2w, H, W, near=0.0, far=3.14):
    cam = ref.pinhole_camera.PinholeCamera(W, H, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    pose = ref.camera_pose.CameraPose.from_camera_to_world(c2w.astype(np.float64))
    cap = ref.captures.BasePinholeCapture(cam, pose)
    cap.near, cap.far = {"bkg": near}, {"bkg": far}
    return cap


def _np(x):
    return x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def _reference_human_net(ref):
    """The reference's HumanNeRF with per-frame SMPL parameters on the CPU, assembled as models/human_nerf.py:31-90 does
    (the hard-coded SMPL pickle path is licence-gated and absent: a synthetic SMPL-shaped pickle instead)."""
    torch.manual_seed(1)
    net = _quiet(ref.human_nerf.HumanNeRF, ref_opts.default_opt(num_offset_nets=1))
    pose, betas, align = T._vf_inputs()
    P = torch.nn.Parameter
    net.poses, net.betas, net.alignments, net.scale = P(torch.from_numpy(pose)), P(torch.from_numpy(betas)), P(torch.from_numpy(align[None])), 0.4
    pk = os.path.join(tempfile.mkdtemp(), "SMPL_NEUTRAL.pkl")
    synth_smpl.write_pickle(pk, 0)
    net.body_model = ref.smpl.SMPL(pk, gender="neutral", device=torch.device("cpu"))
    da = torch.zeros(24, 3)
    da[1, 2], da[2, 2] = 1.0, -1.0
    net.da_smpl = P(da.reshape(1, -1), requires_grad=False)
    return net


def main():
    torch.set_num_threads(1)                 # the tests compare on one thread (tests/test_oracle_vs_reference.py)
    ref = ref_import.load()
    g = {}

    # rays
    H, W = 12, 20
    K, c2w = T._camera(H, W)
    cap = _cap(ref, K, c2w, H, W)
    g["rays.K"], g["rays.c2w"] = _np(cap.intrinsic_matrix), _np(cap.cam_pose.camera_to_world)
    xy = np.argwhere(np.ones((H, W)))[:, ::-1]
    g["rays.o"], g["rays.d"] = (_np(a) for a in ref.ray_utils.shot_rays(cap, xy))
    g["rays.o_all"], g["rays.d_all"] = (_np(a) for a in ref.ray_utils.shot_all_rays(cap))

    # sampling / compositing
    o, d, near, far, raw, S, N = T._sampling_inputs()
    batch = {"origin": o, "direction": d, "near": near, "far": far}
    p, v, z = ref.ray_utils.ray_to_samples(batch, S)
    g["samp.p"], g["samp.v"], g["samp.z"] = _np(p), _np(v), _np(z)
    out = ref.render_utils.raw2outputs(raw, z, d, white_bkg=True)
    for i, a in enumerate(out):
        g[f"samp.out{i}"] = _np(a)
    p, _, z2 = ref.ray_utils.ray_to_importance_samples(batch, z, out[3], N)
    g["samp.imp_p"], g["samp.imp_z"] = _np(p), _np(z2)
    torch.manual_seed(5)
    g["samp.z_perturb"] = _np(ref.ray_utils.ray_to_samples(batch, S, perturb=1.0)[2])

    # networks
    torch.manual_seed(1)
    coarse, fine = ref.vanilla.build_nerf(ref_opts.default_opt())
    human, _ = ref.vanilla.build_nerf(ref_opts.default_opt(posenc="rotate"))
    pts, views = T._net_inputs()
    for name, net in (("coarse", coarse), ("fine", fine), ("human", human)):
        with torch.no_grad():
            g[f"nets.{name}"] = _np(net(pts, views))
        g[f"nets.{name}.checksum"] = T._checksum(net)

    # near / far
    o, d, V = T._near_far_inputs()
    g["nf.n"], g["nf.f"] = ref.ray_utils.geometry_guided_near_far(o, d, V, 0.1)
    n, f = ref.ray_utils.geometry_guided_near_far(torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(V), 0.1)
    g["nf.n_torch"], g["nf.f_torch"] = _np(n), _np(f)

    # SMPL
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "SMPL_NEUTRAL.pkl")
        synth_smpl.write_pickle(path)
        body = ref.smpl.SMPL(path, gender="neutral", device=torch.device("cpu"))
    pose, betas = T._smpl_inputs()
    v_r, T_r = body.verts_transformations(pose, betas, concat_joints=True)
    g["smpl.v"], g["smpl.T"] = _np(v_r[0])[T._rows(v_r.shape[1])], _np(T_r[0])[T._rows(T_r.shape[1])]
    verts, joints = body(pose, betas, return_joints=True)
    verts = _np(verts).reshape(-1, 3)
    g["smpl.verts"], g["smpl.joints"] = verts[T._rows(verts.shape[0])], _np(joints).reshape(-1, 3)

    # warp
    pts, bd, faces6 = T._warp_inputs()
    c, dd, cl = ref.ray_utils.warp_samples_to_canonical(pts, bd["verts"], faces6, bd["Ts"])
    g["warp.c"], g["warp.d"], g["warp.cl"] = _np(c), _np(dd), _np(cl)

    # render_vanilla
    torch.manual_seed(1)
    coarse, fine = ref.vanilla.build_nerf(ref_opts.default_opt())
    H, W = 6, 9
    K, c2w = T._camera(H, W)
    cap = _cap(ref, K, c2w, H, W)
    g["rv.K"], g["rv.c2w"] = _np(cap.intrinsic_matrix), _np(cap.cam_pose.camera_to_world)
    rgb, dep = _quiet(ref.render_utils.render_vanilla, coarse, cap, fine_net=fine, rays_per_batch=32, samples_per_ray=16,
                      importance_samples_per_ray=8, return_depth=True)
    g["rv.rgb"], g["rv.depth"] = _np(rgb), _np(dep)

    # human / hybrid renderers
    torch.manual_seed(1)
    net = _quiet(ref.human_nerf.HumanNeRF, ref_opts.default_opt())
    T._boost(net)
    g["human.checksum"] = T._checksum(T._human_parts(net))
    bd, bd2, H, W, K, c2w = T._human_inputs()
    cap = _cap(ref, K, c2w, H, W)
    g["human.K"], g["human.c2w"] = _np(cap.intrinsic_matrix), _np(cap.cam_pose.camera_to_world)
    faces, geo = bd["faces"], bd["geo_threshold"]
    for can in (True, False):
        r, dd, a = _quiet(ref.render_utils.render_smpl_nerf, net, cap, bd["verts"], faces, bd["Ts"], rays_per_batch=32,
                          samples_per_ray=12, render_can=can, geo_threshold=geo, return_depth=True, return_mask=True,
                          interval_comp=0.7)
        g[f"human.smpl{int(can)}.rgb"], g[f"human.smpl{int(can)}.depth"], g[f"human.smpl{int(can)}.acc"] = _np(r), _np(dd), _np(a)
    r, dd = _quiet(ref.render_utils.render_hybrid_nerf, net, cap, bd["verts"], faces, bd["Ts"], rays_per_batch=32,
                   samples_per_ray=12, importance_samples_per_ray=8, geo_threshold=geo, return_depth=True)
    g["human.hybrid.rgb"], g["human.hybrid.depth"] = _np(r), _np(dd)
    r, dd = _quiet(ref.render_utils.render_hybrid_nerf_multi_persons, net, cap, [net, net], [bd["verts"], bd2["verts"]],
                   [faces, faces], [bd["Ts"], bd2["Ts"]], rays_per_batch=32, samples_per_ray=12,
                   importance_samples_per_ray=8, geo_threshold=geo, return_depth=True)
    g["human.multi.rgb"], g["human.multi.depth"] = _np(r), _np(dd)

    # HumanNeRF state dict (names, shapes, checksums and a few leading values of every tensor)
    torch.manual_seed(11)
    r = _quiet(ref.human_nerf.HumanNeRF, ref_opts.default_opt(num_offset_nets=2))
    sd = r.state_dict()
    g["sd.keys"] = np.array(list(sd.keys()))
    g["sd.shapes"] = np.array([",".join(str(s) for s in t.shape) for t in sd.values()])
    g["sd.sums"] = np.array([float(t.double().sum()) for t in sd.values()])
    g["sd.head"] = np.stack([np.pad(_np(t).reshape(-1)[:4].astype(np.float64), (0, max(0, 4 - t.numel()))) for t in sd.values()])

    # vertex_forward and its gradients
    net = _reference_human_net(ref)
    w_r, T_r = net.vertex_forward(0)
    g1, g2 = T._vertex_cotangents(T_r.shape, w_r.shape)
    ((T_r * g1).sum() + (w_r * g2).sum()).backward()
    r = T._rows(w_r.shape[1])
    g["vf.w"], g["vf.T"] = _np(w_r)[:, r], _np(T_r)[:, r]
    g["vf.g_poses"], g["vf.g_betas"], g["vf.g_align"] = _np(net.poses.grad), _np(net.betas.grad), _np(net.alignments.grad[0])

    # differentiable warp
    P, bd, V, F, Tt = T._diff_warp_inputs()
    Ti, f_id, _ = ref.ray_utils.warp_samples_to_canonical_diff(P, V, F, Tt)
    g["dw.Ti"], g["dw.f_id"] = _np(Ti), _np(f_id)

    # tests/test_host.py: state-dict names, OffsetNet, Embedder / NeRF module interface
    torch.manual_seed(1)
    rc, _ = ref.vanilla.build_nerf(ref_opts.default_opt())
    g["host.nerf_keys"] = np.array(list(rc.state_dict().keys()))
    for st in ("linear", "tanh", "no"):
        torch.manual_seed(3)
        net = ref.vanilla.build_offset_net(ref_opts.default_opt(num_offset_nets=1, offset_scale=0.7, offset_scale_type=st))
        g[f"host.offset.{st}.checksum"] = T._checksum(net)
        x = H_inputs_offset()
        y = net(x)
        y.square().sum().backward()
        g[f"host.offset.{st}.y"] = _np(y)
        for k, q in net.named_parameters():
            g[f"host.offset.{st}.grad.{k}"] = T._grad_summary(q.grad)
    for pe in ("posenc", "rotate"):
        torch.manual_seed(2)
        theirs, _ = ref.vanilla.build_nerf(ref_opts.default_opt(posenc=pe))
        for e in (theirs.pos_pe, theirs.dir_pe):
            if hasattr(e, "bvals"):
                e.bvals = e.bvals.cpu()                # the reference parks them on the GPU whenever one is visible
        x, v = H_inputs_module()
        with torch.no_grad():
            g[f"host.module.{pe}.pos_pe"], g[f"host.module.{pe}.dir_pe"] = _np(theirs.pos_pe(x)), _np(theirs.dir_pe(v))
            g[f"host.module.{pe}.joiner"] = _np(theirs(x, v))

    np.savez_compressed(OUT, **{k: np.asarray(v) for k, v in g.items()})
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(g)} arrays")


if __name__ == "__main__":
    main()
