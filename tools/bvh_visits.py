"""CPU emulation of the warp stage's packet BVH traversal (neuman_b200/csrc/warp.cu: LBVH build, bvh_nearest_face): counts
internal-node visits, triangle tests and stack pops per 32-lane packet for the packet shapes of k_warp_nearest, on the
hit rays of the cfg4/cfg5 body.
python tools/bvh_visits.py"""
import sys, os
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neuman_b200 import synthetic
from oracle import synth_smpl, neuman_oracle as no

def expand(v):
    v = v.astype(np.uint64)
    v = (v * 0x00010001) & 0xFF0000FF
    v = (v * 0x00000101) & 0x0F00F00F
    v = (v * 0x00000011) & 0xC30C30C3
    v = (v * 0x00000005) & 0x49249249
    return v

def build(verts, faces):
    tri = verts[faces]                                # [F,3,3]
    lo, hi = verts.min(0), verts.max(0)
    c = (tri.mean(1) - lo) / np.maximum(hi - lo, 1e-20)
    q = np.clip((c * 1024).astype(np.int64), 0, 1023)
    m = (expand(q[:, 0]) << 2) | (expand(q[:, 1]) << 1) | expand(q[:, 2])
    keys = (m.astype(np.uint64) << np.uint64(32)) | np.arange(len(faces), dtype=np.uint64)
    keys = np.sort(keys)
    n = len(keys)
    leaf_face = (keys & np.uint64(0xffffffff)).astype(np.int64)
    kl = [int(k) for k in keys]
    def delta(i, j):
        if j < 0 or j >= n: return -1
        x = kl[i] ^ kl[j]
        return 64 - x.bit_length()
    children = np.zeros((n - 1, 2), np.int64); parent = np.full(2 * n - 1, -1, np.int64)
    for i in range(n - 1):
        d = 1 if delta(i, i + 1) - delta(i, i - 1) >= 0 else -1
        dmin = delta(i, i - d)
        lmax = 2
        while delta(i, i + lmax * d) > dmin: lmax <<= 1
        l = 0; t = lmax >> 1
        while t >= 1:
            if delta(i, i + (l + t) * d) > dmin: l += t
            t >>= 1
        j = i + l * d
        dn = delta(i, j)
        s = 0; t = l
        while True:
            t = (t + 1) >> 1
            if delta(i, i + (s + t) * d) > dn: s += t
            if t <= 1: break
        g = i + s * d + min(d, 0)
        left = n - 1 + g if min(i, j) == g else g
        right = n - 1 + g + 1 if max(i, j) == g + 1 else g + 1
        children[i] = (left, right); parent[left] = i; parent[right] = i
    blo = np.zeros((2 * n - 1, 3), np.float32); bhi = np.zeros((2 * n - 1, 3), np.float32)
    t = tri[leaf_face]
    blo[n - 1:] = t.min(1); bhi[n - 1:] = t.max(1)
    # refit: process internal nodes in order of decreasing depth
    depth = np.zeros(2 * n - 1, np.int64)
    order = [0]
    for node in order:
        if node < n - 1:
            for ch in children[node]:
                depth[ch] = depth[node] + 1; order.append(int(ch))
    for node in reversed(order):
        if node < n - 1:
            a, b = children[node]
            blo[node] = np.minimum(blo[a], blo[b]); bhi[node] = np.maximum(bhi[a], bhi[b])
    return dict(n=n, children=children, lo=blo, hi=bhi, leaf_face=leaf_face, tri=tri.astype(np.float32), depth=depth)

def closest_d2(p, tri):
    """p [L,3], tri [3,3] -> squared distance [L] (Ericson regions), float32."""
    a, b, c = tri
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = ap @ ab, ap @ ac
    bp = p - b; d3, d4 = bp @ ab, bp @ ac
    cp = p - c; d5, d6 = cp @ ab, cp @ ac
    vc = d1 * d4 - d3 * d2; vb = d5 * d2 - d1 * d6; va = d3 * d6 - d5 * d4
    out = np.empty_like(p)
    done = np.zeros(len(p), bool)
    def put(mask, val):
        nonlocal done
        m = mask & ~done
        out[m] = val[m] if val.ndim == 2 else val
        done |= m
    put((d1 <= 0) & (d2 <= 0), np.broadcast_to(a, p.shape))
    put((d3 >= 0) & (d4 <= d3), np.broadcast_to(b, p.shape))
    with np.errstate(all="ignore"):
        put((vc <= 0) & (d1 >= 0) & (d3 <= 0), a + ab * (d1 / (d1 - d3))[:, None])
        put((d6 >= 0) & (d5 <= d6), np.broadcast_to(c, p.shape))
        put((vb <= 0) & (d2 >= 0) & (d6 <= 0), a + ac * (d2 / (d2 - d6))[:, None])
        put((va <= 0) & ((d4 - d3) >= 0) & ((d5 - d6) >= 0), b + (c - b) * ((d4 - d3) / ((d4 - d3) + (d5 - d6)))[:, None])
        den = 1.0 / (va + vb + vc)
        put(np.ones(len(p), bool), a + ab * (vb * den)[:, None] + ac * (vc * den)[:, None])
    e = out - p
    return (e * e).sum(1)

def box_d2(B, node, p):
    d = np.maximum(np.maximum(B["lo"][node] - p, p - B["hi"][node]), 0)
    return (d * d).sum(1)

def traverse(B, p, seed_best=None):
    """packet traversal as in bvh_nearest_face; returns (best_f, visits_internal, leaf_tests, pops)"""
    n = B["n"]; L = len(p)
    best = np.full(L, np.float32(3.4e38)) if seed_best is None else seed_best.copy()
    best_f = np.full(L, 2**31 - 1)
    stack = []; node = 0
    vi = vl = pops = 0
    while True:
        if node >= n - 1:
            f = B["leaf_face"][node - (n - 1)]
            d2 = closest_d2(p, B["tri"][f])
            upd = (d2 < best) | ((d2 == best) & (f < best_f))
            best = np.where(upd, d2, best); best_f = np.where(upd, f, best_f)
            vl += 1; node = -1
        else:
            vi += 1
            l, r = B["children"][node]
            dl, dr = box_d2(B, l, p), box_d2(B, r, p)
            lim = best * np.float32(1.00001)
            nl, nr = (dl <= lim).any(), (dr <= lim).any()
            lf = 2 * (dl <= dr).sum() >= L
            if nl and nr:
                stack.append(r if lf else l); node = l if lf else r
            else:
                node = l if nl else (r if nr else -1)
        if node < 0:
            found = False
            while stack:
                cand = stack.pop(); pops += 1
                if (box_d2(B, cand, p) <= best * np.float32(1.00001)).any():
                    node = cand; found = True; break
            if not found: break
    return best_f, vi, vl, pops, best

if __name__ == "__main__":
    import torch
    b = synth_smpl.random_body(seed=1, scale=0.45, center=(0.1, 0.0, 0.3))
    verts, faces = np.asarray(b["verts"], np.float32), np.asarray(b["faces"], np.int64)
    B = build(verts, faces)
    H, W = 720, 1280
    K, c2w = synthetic.camera(H, W, seed=1)
    o, d = no.shot_all_rays(K, c2w, H, W)
    o = np.asarray(o, np.float32); d = np.asarray(d, np.float32)
    # subsample rays on a grid of 4-neighbourhoods: take blocks of 8 consecutive pixels every ~ 997 pixels
    rng = np.random.default_rng(0)
    starts = rng.choice(H * W // 8, 6000, replace=False) * 8
    idx = (starts[:, None] + np.arange(8)[None]).reshape(-1)
    nr, fr = no.geometry_guided_near_far(torch.from_numpy(o[idx]), torch.from_numpy(d[idx]), torch.from_numpy(verts), b["geo_threshold"])
    nr, fr = np.asarray(nr).reshape(-1), np.asarray(fr).reshape(-1)
    hit = nr < fr
    print("hit frac", hit.mean(), "hits", hit.sum())
    S = 128
    t = np.linspace(0, 1, S, dtype=np.float32)
    hi = np.flatnonzero(hit)
    # groups of 4 adjacent hit rays (same 8-block)
    blocks = {}
    for k in hi: blocks.setdefault(k // 8, []).append(k)
    groups = [v[:4] for v in blocks.values() if len(v) >= 4][:60]
    print("groups", len(groups))
    def pts_of(k):
        z = nr[k] * (1 - t) + fr[k] * t
        return o[idx[k]][None] + d[idx[k]][None] * z[:, None]
    stats = {"ray32": [], "4x8": [], "single": []}
    dists = []
    for g in groups:
        P = np.stack([pts_of(k) for k in g])        # [4,S,3]
        # 1 ray x 32 samples
        for sg in range(0, S, 32):
            bf, vi, vl, pops, best = traverse(B, P[0, sg:sg + 32]); stats["ray32"].append((vi, vl, pops)); dists.append(np.sqrt(best))
        for sg in range(0, S, 8):
            bf, vi, vl, pops, best = traverse(B, P[:, sg:sg + 8].reshape(-1, 3)); stats["4x8"].append((vi, vl, pops))
        for s in range(0, S, 16):
            bf, vi, vl, pops, best = traverse(B, P[0, s:s + 1]); stats["single"].append((vi, vl, pops))
    for k, v in stats.items():
        v = np.array(v, float); print(k, "internal, leaves, pops per packet:", v.mean(0), "max", v.max(0))
    dists = np.concatenate(dists); print("dist mean/median/max", dists.mean(), np.median(dists), dists.max(), "thr", b["geo_threshold"])
