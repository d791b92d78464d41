"""Bit-for-bit comparison of the tensor-core MLP forward and backward chain and the frame drivers between two builds of the
library.

    python tools/fwd_digest.py dump OUT.json [--root TREE]     # run TREE's library (default: this tree) on seeded inputs
    python tools/fwd_digest.py compare A.json B.json           # exit 1 unless every record is identical

`dump` runs the tensor-core forward on seeded inputs and records a SHA-256 of every output buffer: the training forward's raw,
activation stash (st_x, st_f, st_v) and sign words, the backward chain's gradient planes (nm_mlp_backward on that stash with a
seeded d_raw and a fixed loss scale: g_pre, g_f, g_v), and the inference raw in per-sample, per-ray-view and fused ray modes,
for view-dependent nets (posenc and rotate), a view-independent net (no st_f / st_v / g_f / g_v, 8 sign-word planes) and a
NeRF-T net ([n,4] points; no fused ray mode, which NeRF-T slots do not take).  The weight-gradient GEMM (nm_dw_gemm) is not
recorded: it sums across CTAs with red.global.add, so its output's last bits vary from run to run.  Sizes
cover ragged tiles, several waves of the persistent grid and a frame-sized ray chunk.  Its frames section renders with
every driver (vanilla coarse-only and coarse + fine, smpl_nerf canonical and posed, hybrid, multi-person with 2 and 3
actors), each with host and device output, a pixel range and a pixel list, the default chunk and a ragged one, and
records the SHA-256 of rgb, depth and acc with the call's library launch count and render statistics.  Run it once from
each build's tree (each loads its own libneuman_b200.so) and compare the two files."""
import argparse
import hashlib
import json
import os
import sys


def _digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def dump(out, root):
    sys.path.insert(0, root)
    import torch
    import neuman_b200 as nb
    from neuman_b200 import _lib, ops
    from neuman_b200.ops import _p
    from oracle import scenes
    assert os.path.dirname(os.path.abspath(_lib.LIB_PATH)).startswith(os.path.abspath(root)), _lib.LIB_PATH
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    coarse, _ = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False), 1)
    human, _ = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False, posenc="rotate"), 2)
    noview, _ = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False, use_viewdirs=False), 3)
    nerft, _ = scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False, raw_pos_dim=4), 4)
    T = 128 * torch.cuda.get_device_properties(0).multi_processor_count
    res = {"lib": _lib.LIB_PATH}
    for name, j in (("coarse", coarse.to(dev)), ("human", human.to(dev)), ("noview", noview.to(dev)), ("nerft", nerft.to(dev))):
        view, time = name != "noview", name == "nerft"
        ctx = ops._ctx_for(torch.empty(1, device=dev))
        slot = ops.net_slot(j, ctx)
        for n in (1, 129, 4173, 3 * T - 5):
            g = torch.Generator(device=dev).manual_seed(n)
            pts = torch.randn(n, 3, device=dev, generator=g) * 1.5
            views = torch.nn.functional.normalize(torch.randn(n, 3, device=dev, generator=g), dim=-1)
            if time:                                 # (x, y, z, t), t in [0, 1)
                pts = torch.cat([pts, torch.rand(n, 1, device=dev, generator=g)], dim=1).contiguous()
            # training forward, per-sample views
            raw = torch.empty(n, 4, device=dev)
            sx = torch.empty(8, n, 256, device=dev, dtype=torch.float16)
            sf = torch.empty(n, 256, device=dev, dtype=torch.float16)
            sv = torch.empty(n, 128, device=dev, dtype=torch.float16)
            sm = torch.empty(9 if view else 8, n, 8, device=dev, dtype=torch.int32)
            ctx.check(ctx.lib.nm_mlp_forward_train(ctx.h, slot, _p(pts), _p(views), n, 0, _p(raw), _p(sx), _p(sf), _p(sv),
                                                   _p(sm), ctx.stream()))
            torch.cuda.synchronize()
            outs = (("raw", raw), ("st_x", sx), ("st_f", sf), ("st_v", sv), ("st_m", sm)) if view else \
                (("raw", raw), ("st_x", sx), ("st_m", sm))
            for k, v in outs:
                res[f"{name}/train/n={n}/{k}"] = _digest(v)
            # backward chain on that stash, loss scale 2^6 (max |d_raw| * S about 256, as autograd picks it)
            d_raw = torch.randn(n, 4, device=dev, generator=g)
            scale = torch.full((1,), 64.0, device=dev)
            gp = torch.empty(8, n, 256, device=dev, dtype=torch.float16)
            gf = torch.empty(n, 256, device=dev, dtype=torch.float16) if view else None
            gv = torch.empty(n, 128, device=dev, dtype=torch.float16) if view else None
            ctx.check(ctx.lib.nm_mlp_backward(ctx.h, slot, _p(d_raw), _p(scale), n, _p(sv if view else None), _p(sm), _p(gp),
                                              _p(gf), _p(gv), ctx.stream()))
            torch.cuda.synchronize()
            for k, v in (("g_pre", gp), ("g_f", gf), ("g_v", gv)) if view else (("g_pre", gp),):
                res[f"{name}/backward/n={n}/{k}"] = _digest(v)
            # inference, per-sample views and one view row per 7 samples (n rounded down to a multiple of 7)
            for group in (0,) if time else (0, 7):
                m = n if group == 0 else n - n % group
                if m == 0:
                    continue
                vrows = views if group == 0 else views[: m // group].contiguous()
                raw = torch.empty(m, 4, device=dev)
                ctx.check(ctx.lib.nm_mlp_forward(ctx.h, slot, _lib.NM_MLP_TC_F16, _p(pts), _p(vrows), m, group, _p(raw),
                                                 ctx.stream()))
                torch.cuda.synchronize()
                res[f"{name}/infer/n={m}/group={group}/raw"] = _digest(raw)
        # fused ray mode (pts = o + d z), up to a frame's chunk of 32768 rays x 256 samples
        for R, S in () if time else ((1, 1), (33, 33), (97, 128), (4096, 128), (32768, 256)):
            g = torch.Generator(device=dev).manual_seed(R * 1000 + S)
            o = torch.randn(R, 3, device=dev, generator=g) * 0.3
            d = torch.nn.functional.normalize(torch.randn(R, 3, device=dev, generator=g), dim=-1)
            z = torch.sort(torch.rand(R, S, device=dev, generator=g) * 3.14, dim=-1)[0].contiguous()
            raw = ops.mlp_forward_rays(j, o, d, z, mode=_lib.NM_MLP_TC_F16)
            torch.cuda.synchronize()
            res[f"{name}/rays/R={R}/S={S}/raw"] = _digest(raw)
    frames(res, dev)
    _lib.Context.get(0).range_check()
    with open(out, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
    print(f"{len(res) - 1} digests of {res['lib']} -> {out}")


def frames(res, dev):
    import torch
    import neuman_b200 as nb
    from neuman_b200 import _lib, render, sharding
    from oracle import scenes, synth_smpl
    ctx = _lib.Context.get(0)
    coarse, fine = (m.to(dev) for m in scenes.seed_nets(nb.build_nerf, nb.default_opt(use_cuda=False), 1))
    torch.manual_seed(1)
    human = nb.HumanNeRF(nb.default_opt(use_cuda=False))
    scenes.boost_density(human.coarse_human_net)
    human = human.to(dev)
    H, W = 180, 240                                  # 43200 rays: two default chunks of the vanilla and hybrid drivers
    K, c2w = scenes.camera(H, W, focal=200.0, seed=0)
    cap = nb.SimpleCapture(K, c2w, H, W, 0.0, 3.14)
    bodies = [synth_smpl.random_body(seed=s, center=c) for s, c in ((1, (0.1, 0.0, 0.3)), (4, (-0.15, 0.0, 0.5)),
                                                                     (7, (0.35, 0.05, 0.7)))]
    b, geo = bodies[0], bodies[0]["geo_threshold"]

    def multi(k):
        v, f, t = ([x[key] for x in bodies[:k]] for key in ("verts", "faces", "Ts"))

        def run(pix0, n, host_out, chunk, pixels):
            return render._hybrid(human, [human] * k, cap, v, f, t, 32, 32, True, geo, True, pix0, n, host_out, chunk, pixels=pixels)
        return run
    drivers = {
        "vanilla_coarse": (lambda **kw: render.render_vanilla_range(coarse, cap, None, 32, 0, **kw), render.CHUNK),
        "vanilla_fine": (lambda **kw: render.render_vanilla_range(coarse, cap, fine, 32, 32, **kw), render.CHUNK),
        "smpl_canonical": (lambda **kw: render.render_smpl_nerf_range(human, cap, b["verts"], b["faces"], b["Ts"], 32, True, True,
                                                                      geo, 0.7, **kw), render.SMPL_CHUNK),
        "smpl_posed": (lambda **kw: render.render_smpl_nerf_range(human, cap, b["verts"], b["faces"], b["Ts"], 32, True, False,
                                                                  geo, 0.7, **kw), render.SMPL_CHUNK),
        "hybrid": (lambda **kw: render.render_hybrid_nerf_range(human, cap, b["verts"], b["faces"], b["Ts"], 32, 32, True, geo,
                                                                **kw), render.CHUNK),
        "multi2": (multi(2), render.CHUNK),
        "multi3": (multi(3), render.CHUNK),
    }
    pixel_list = torch.from_numpy(sharding.tile_pixels(H, W, 1, 3)).to(dev)
    for name, (fn, default_chunk) in drivers.items():
        for host_out in (True, False):
            for where, pix0, n, pixels in (("range", 1234, H * W - 1801, None), ("list", 0, None, pixel_list)):
                for chunk in (default_chunk, 777):
                    key = f"frames/{name}/host_out={int(host_out)}/{where}/chunk={chunk}"
                    l0 = ctx.launch_count()
                    outs = fn(pix0=pix0, n=n, host_out=host_out, chunk=chunk, pixels=pixels)
                    torch.cuda.synchronize()
                    res[key + "/launches"] = ctx.launch_count() - l0
                    res[key + "/stats"] = ctx.render_stats()
                    for plane, t in zip(("rgb", "depth", "acc"), outs):
                        res[f"{key}/{plane}"] = _digest(t)


def compare(a, b):
    A, B = (json.load(open(p)) for p in (a, b))
    keys = sorted((set(A) | set(B)) - {"lib"})
    bad = [k for k in keys if A.get(k) != B.get(k)]
    for k in bad:
        print("DIFFERENT", k)
    print(f"{len(keys) - len(bad)} of {len(keys)} records identical ({A['lib']} vs {B['lib']})")
    return 1 if bad else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("cmd", choices=["dump", "compare"])
    ap.add_argument("files", nargs="+")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    a = ap.parse_args()
    if a.cmd == "dump":
        dump(a.files[0], os.path.abspath(a.root))
    else:
        sys.exit(compare(*a.files))
