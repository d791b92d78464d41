"""TEST INFRASTRUCTURE ONLY (oracle) -- float64 restatement of the three libigl calls on the NeuMan
hot path.  **Parity unpinned**: libigl 2.2.1 (environment.yml:13) is a third-party C++ dependency
that is not part of the reference tree, and the reference holds no golden vectors
at this boundary (SURVEY.md §8c).  This file restates the *published* semantics of

  igl.point_mesh_squared_distance(P, V, F) -> (sqrD, I, C)   call site utils/ray_utils.py:53
  igl.barycentric_coordinates_tri(P, A, B, C) -> L            call site utils/ray_utils.py:55
  igl.signed_distance(P, V, F) -> (S, I, C)                   call sites utils/ray_utils.py:70,
                                                              trainers/human_nerf_trainer.py:310,326

i.e. exact Euclidean closest point on a triangle soup (vertex / edge / face Voronoi regions,
Ericson, "Real-Time Collision Detection" §5.1.5), arg-min over faces (lowest face index wins exact
ties), barycentric coordinates of a point with respect to (A, B, C) in that vertex order, and the
sign of the distance from the angle-weighted pseudo-normal at the closest feature.

The search is exhaustive but pruned with an *exact* bound (a triangle whose bounding sphere is
farther than the nearest vertex cannot hold the closest point), so results equal brute force.
"""
import numpy as np


def _closest_on_triangles(p, a, b, c):
    """p, a, b, c: [n,3] float64 (one triangle per point). Returns closest points [n,3]."""
    ab = b - a
    ac = c - a
    ap = p - a
    d1 = np.einsum("ij,ij->i", ab, ap)
    d2 = np.einsum("ij,ij->i", ac, ap)
    bp = p - b
    d3 = np.einsum("ij,ij->i", ab, bp)
    d4 = np.einsum("ij,ij->i", ac, bp)
    cp = p - c
    d5 = np.einsum("ij,ij->i", ab, cp)
    d6 = np.einsum("ij,ij->i", ac, cp)
    vc = d1 * d4 - d3 * d2
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4

    with np.errstate(divide="ignore", invalid="ignore"):
        # face interior (default)
        denom = 1.0 / (va + vb + vc)
        v = vb * denom
        w = vc * denom
        out = a + ab * v[:, None] + ac * w[:, None]
        # edge BC
        m = (va <= 0) & ((d4 - d3) >= 0) & ((d5 - d6) >= 0)
        t = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        out = np.where(m[:, None], b + (c - b) * t[:, None], out)
        # edge AC
        m = (vb <= 0) & (d2 >= 0) & (d6 <= 0)
        t = d2 / (d2 - d6)
        out = np.where(m[:, None], a + ac * t[:, None], out)
        # vertex C
        m = (d6 >= 0) & (d5 <= d6)
        out = np.where(m[:, None], c, out)
        # edge AB
        m = (vc <= 0) & (d1 >= 0) & (d3 <= 0)
        t = d1 / (d1 - d3)
        out = np.where(m[:, None], a + ab * t[:, None], out)
        # vertex B
        m = (d3 >= 0) & (d4 <= d3)
        out = np.where(m[:, None], b, out)
        # vertex A
        m = (d1 <= 0) & (d2 <= 0)
        out = np.where(m[:, None], a, out)
    return out


def point_mesh_squared_distance(P, V, F, chunk=1024):
    """Restates igl.point_mesh_squared_distance (utils/ray_utils.py:53). float64 throughout."""
    P = np.asarray(P, dtype=np.float64).reshape(-1, 3)
    V = np.asarray(V, dtype=np.float64)
    F = np.asarray(F)[:, :3].astype(np.int64)
    A, B, C = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    cen = (A + B + C) / 3.0
    rad = np.sqrt(np.maximum(np.maximum(((A - cen) ** 2).sum(1), ((B - cen) ** 2).sum(1)),
                             ((C - cen) ** 2).sum(1)))
    n = P.shape[0]
    sqrD = np.empty(n)
    I = np.empty(n, dtype=np.int64)
    Cl = np.empty((n, 3))
    v2 = (V ** 2).sum(1)
    c2 = (cen ** 2).sum(1)
    for s in range(0, n, chunk):
        p = P[s:s + chunk]
        p2 = (p ** 2).sum(1)
        # upper bound: nearest vertex
        dv = np.sqrt(np.maximum(p2[:, None] - 2.0 * p @ V.T + v2[None, :], 0.0)).min(1)
        dc = np.sqrt(np.maximum(p2[:, None] - 2.0 * p @ cen.T + c2[None, :], 0.0))
        cand = (dc - rad[None, :]) <= (dv[:, None] * (1 + 1e-6) + 1e-9)
        pi, fi = np.nonzero(cand)          # sorted by point, then by face index
        cl = _closest_on_triangles(p[pi], A[fi], B[fi], C[fi])
        d2 = ((cl - p[pi]) ** 2).sum(1)
        # segmented arg-min, first occurrence wins
        starts = np.flatnonzero(np.r_[True, pi[1:] != pi[:-1]])
        seg_min = np.minimum.reduceat(d2, starts)
        seg_id = np.cumsum(np.r_[True, pi[1:] != pi[:-1]]) - 1
        is_min = d2 == seg_min[seg_id]
        idx = np.flatnonzero(is_min)
        first = idx[np.r_[True, seg_id[idx][1:] != seg_id[idx][:-1]]]
        rows = pi[first]
        sqrD[s + rows] = d2[first]
        I[s + rows] = fi[first]
        Cl[s + rows] = cl[first]
    return sqrD, I, Cl


def barycentric_coordinates_tri(P, A, B, C):
    """Restates igl.barycentric_coordinates_tri (utils/ray_utils.py:55): sub-triangle areas
    over the triangle area (signed through the triangle normal), L[:,k] weights vertex k."""
    P, A, B, C = (np.asarray(x, dtype=np.float64) for x in (P, A, B, C))
    n = np.cross(B - A, C - A)
    nn = np.einsum("ij,ij->i", n, n)
    la = np.einsum("ij,ij->i", n, np.cross(C - B, P - B)) / nn
    lb = np.einsum("ij,ij->i", n, np.cross(A - C, P - C)) / nn
    lc = 1.0 - la - lb
    return np.stack([la, lb, lc], axis=1)


def _pseudonormals(V, F):
    A, B, C = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    fn = np.cross(B - A, C - A)
    fn /= np.maximum(np.linalg.norm(fn, axis=1, keepdims=True), 1e-300)
    vn = np.zeros_like(V)

    def ang(u, v):
        cu = np.einsum("ij,ij->i", u, v) / np.maximum(
            np.linalg.norm(u, axis=1) * np.linalg.norm(v, axis=1), 1e-300)
        return np.arccos(np.clip(cu, -1, 1))
    np.add.at(vn, F[:, 0], fn * ang(B - A, C - A)[:, None])
    np.add.at(vn, F[:, 1], fn * ang(C - B, A - B)[:, None])
    np.add.at(vn, F[:, 2], fn * ang(A - C, B - C)[:, None])
    edge_n = {}
    for f, (i, j, k) in enumerate(F):
        for e in ((i, j), (j, k), (k, i)):
            key = (min(e), max(e))
            edge_n[key] = edge_n.get(key, 0) + fn[f]
    return fn, vn, edge_n


def signed_distance(P, V, F):
    """Restates igl.signed_distance with the pseudo-normal sign (utils/ray_utils.py:70).
    Returns (S, I, C)."""
    P = np.asarray(P, dtype=np.float64).reshape(-1, 3)
    V = np.asarray(V, dtype=np.float64)
    F = np.asarray(F)[:, :3].astype(np.int64)
    sqrD, I, Cl = point_mesh_squared_distance(P, V, F)
    fn, vn, edge_n = _pseudonormals(V, F)
    L = barycentric_coordinates_tri(Cl, V[F[I, 0]], V[F[I, 1]], V[F[I, 2]])
    eps = 1e-9
    N = fn[I].copy()
    on = L > eps
    cnt = on.sum(1)
    for r in np.flatnonzero(cnt == 1):
        N[r] = vn[F[I[r], np.argmax(L[r])]]
    for r in np.flatnonzero(cnt == 2):
        ks = np.flatnonzero(on[r])
        i, j = F[I[r], ks[0]], F[I[r], ks[1]]
        N[r] = edge_n[(min(i, j), max(i, j))]
    sgn = np.sign(np.einsum("ij,ij->i", P - Cl, N))
    sgn[sgn == 0] = 1.0
    return sgn * np.sqrt(sqrD), I, Cl
