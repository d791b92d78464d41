"""Exact restatements of the ray-marching stage kernels (csrc/rays.cu, csrc/resample.cu, csrc/composite.cu) for
element-by-element checks.

Those kernels are built with -fmad=false and use only correctly rounded fp32 / fp64 operations (add, mul, div, sqrt,
compare, min / max), except expf in the composite.  So a numpy float32 / float64 restatement in the kernel's own
operation order -- the per-lane partial sums, the butterflies and the Hillis-Steele lane scans included -- gives the
kernel's results bit for bit: raygen, ray_to_samples, near/far (k_near_far and the grouped k_near_far_groups), the cdf
and its inversion (build_cdf / invert_cdf), importance sampling and the merge.

The composite is held to a float64 window instead: `Val` carries, for every intermediate of the kernel, the exact value
`e` (float64) of the same expression and a bound `B` on |kernel - e|, propagated through the kernel's operation order
(each fp32 operation adds at most 2^-24 (|e| + B) + 2^-149; expf at most 2 ulp = 2^-22 |result|).  The windows are per
element, never scaled by a batch maximum.  `f` is a float32 emulation of the same chain (numpy's expf), so the CPU can
show that the window holds the fixed chain and rejects a planted defect.  Everything here runs on the CPU."""
import numpy as np

F32, F64 = np.float32, np.float64
U = 2.0 ** -24                 # fp32 unit roundoff (round to nearest)
TINY = 2.0 ** -149             # absolute rounding error near the underflow range
LANES = 32


def linspace01(i, steps):
    """nm_linspace01 (csrc/nm_internal.cuh): torch.linspace(0, 1, steps)[i] in float32, both halves."""
    i = np.asarray(i)
    if steps <= 1:
        return np.zeros(i.shape, F32)
    step = F32(1.0) / F32(steps - 1)
    lo = i.astype(F32) * step
    hi = F32(1.0) - (steps - 1 - i).astype(F32) * step
    return np.where(i < steps // 2, lo, hi).astype(F32)


# ---------------------------------------------------------------------------------------------
# raygen (k_raygen, invert3x3)
# ---------------------------------------------------------------------------------------------
def invert3x3(m):
    a, b, c, d, e, f, g, h, i = (float(x) for x in np.asarray(m, F64).reshape(-1))
    det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g)
    r = 1.0 / det
    return np.array([(e * i - f * h) * r, (c * h - b * i) * r, (b * f - c * e) * r,
                     (f * g - d * i) * r, (a * i - c * g) * r, (c * d - a * f) * r,
                     (d * h - e * g) * r, (b * g - a * h) * r, (a * e - b * d) * r], F64)


def raygen(K, c2w, W, mode, pix=None, xy=None):
    """(origins, dirs) float32 [n,3] of k_raygen for row-major pixel indices `pix` or integer pairs `xy` [n,2]."""
    Ki = invert3x3(K)
    M = np.asarray(c2w, F64).reshape(-1)
    if xy is not None:
        x, y = np.asarray(xy)[:, 0].astype(F64), np.asarray(xy)[:, 1].astype(F64)
    else:
        pix = np.asarray(pix, np.int64)
        y, x = (pix // W).astype(F64), (pix % W).astype(F64)
    cx = Ki[0] * x + Ki[1] * y + Ki[2]
    cy = Ki[3] * x + Ki[4] * y + Ki[5]
    cz = Ki[6] * x + Ki[7] * y + Ki[8]
    w = [M[4 * k] * cx + M[4 * k + 1] * cy + M[4 * k + 2] * cz + M[4 * k + 3] for k in range(4)]
    wx, wy, wz = w[0] / w[3], w[1] / w[3], w[2] / w[3]
    o = np.array([M[3], M[7], M[11]]).astype(F32)
    if mode == 0:
        f = [wx.astype(F32) - o[0], wy.astype(F32) - o[1], wz.astype(F32) - o[2]]
        nrm = np.sqrt(f[0] * f[0] + f[1] * f[1] + f[2] * f[2])
        d = np.stack([f[0] / nrm, f[1] / nrm, f[2] / nrm], 1)
    else:
        ex, ey, ez = wx - F64(o[0]), wy - F64(o[1]), wz - F64(o[2])
        nrm = np.sqrt(ex * ex + ey * ey + ez * ez)
        d = np.stack([ex / nrm, ey / nrm, ez / nrm], 1).astype(F32)
    return np.broadcast_to(o, d.shape).copy(), d


# ---------------------------------------------------------------------------------------------
# ray_to_samples (k_ray_to_samples)
# ---------------------------------------------------------------------------------------------
def ray_to_samples(o, d, near, far, S, lindisp=False, t_rand=None):
    """(pts [R,S,3], z [R,S]); near / far: [R] arrays or python scalars (the kernel's scalar fallback)."""
    o, d = np.asarray(o, F32), np.asarray(d, F32)
    R = o.shape[0]
    nr = np.broadcast_to(np.asarray(near, F32).reshape(-1, 1), (R, 1))
    fr = np.broadcast_to(np.asarray(far, F32).reshape(-1, 1), (R, 1))
    one = F32(1.0)

    def zval(i):
        t = linspace01(i, S)[None, :]
        if not lindisp:
            return nr * (one - t) + fr * t
        return one / (one / nr * (one - t) + one / fr * t)
    s = np.arange(S)
    z = zval(s)
    if t_rand is not None:
        zl = np.where(s > 0, zval(np.maximum(s - 1, 0)), z)
        zu = np.where(s < S - 1, zval(np.minimum(s + 1, S - 1)), z)
        half = F32(0.5)
        lower = np.where(s > 0, half * (z + zl), z)
        upper = np.where(s < S - 1, half * (zu + z), z)
        u = np.minimum(np.maximum(np.asarray(t_rand, F32), F32(0.01)), one - F32(0.01))
        z = lower + (upper - lower) * u
    z = z.astype(F32)
    pts = o[:, None, :] + d[:, None, :] * z[..., None]
    return pts, z


# ---------------------------------------------------------------------------------------------
# near / far (k_near_far, k_near_far_groups, nm_impl_build_vgroups)
# ---------------------------------------------------------------------------------------------
def thr_sq(geo_threshold):
    thr = F32(geo_threshold)
    return thr, F32(float(thr) * float(thr))


def near_far_exhaustive(o, d, verts, geo_threshold, chunk=256):
    """The per-vertex sphere test of both kernels over every vertex, no cull: near = min(z0 - dz), far = max(z0 + dz)
    over the vertices with disc >= 0; a miss gives (+inf, -inf)."""
    o, d, v = np.asarray(o, F32), np.asarray(d, F32), np.asarray(verts, F32)
    _, thr2 = thr_sq(geo_threshold)
    nears, fars = [], []
    for s in range(0, o.shape[0], chunk):
        oc, dc = o[s:s + chunk, None, :], d[s:s + chunk, None, :]
        ax, ay, az = v[None, :, 0] - oc[..., 0], v[None, :, 1] - oc[..., 1], v[None, :, 2] - oc[..., 2]
        z0 = ax * dc[..., 0] + ay * dc[..., 1] + az * dc[..., 2]
        nrm = np.sqrt(ax * ax + ay * ay + az * az)
        disc = thr2 - (nrm * nrm - z0 * z0)
        hit = disc >= 0
        dz = np.sqrt(np.where(hit, disc, F32(0)))
        nears.append(np.where(hit, z0 - dz, F32(np.inf)).min(1))
        fars.append(np.where(hit, z0 + dz, F32(-np.inf)).max(1))
    return np.concatenate(nears).astype(F32), np.concatenate(fars).astype(F32)


def _expand10(v):
    v = v.astype(np.uint64)
    m = 0xFFFFFFFF
    v = (v * 0x00010001) & 0xFF0000FF & m
    v = (v * 0x00000101) & 0x0F00F00F & m
    v = (v * 0x00000011) & 0xC30C30C3 & m
    v = (v * 0x00000005) & 0x49249249 & m
    return v


def _sphere(p, lo, hi):
    """bbox centre and max distance of the points p [.., n, 3], in the host code's float32 order"""
    half = F32(0.5)
    c = half * (lo + hi)
    q = p - c[..., None, :]
    r2 = (q[..., 0] * q[..., 0] + q[..., 1] * q[..., 1]) + q[..., 2] * q[..., 2]
    return c, np.sqrt(r2.max(-1))


def vertex_groups(verts):
    """nm_impl_build_vgroups: Morton order, groups of 32 (the last padded with its first vertex), one bounding sphere
    per group, and the whole mesh's sphere.  Returns (grouped verts [G,32,3], centres [G,3], radii [G], centre, radius)."""
    hv = np.asarray(verts, F32)
    nv = hv.shape[0]
    lo, hi = hv.min(0), hv.max(0)
    inv = F32(1023.0) / np.maximum(hi - lo, F32(1e-20))
    q = np.minimum(np.maximum((hv - lo) * inv, F32(0)), F32(1023)).astype(np.uint32)
    key = (_expand10(q[:, 0]) << 2) | (_expand10(q[:, 1]) << 1) | _expand10(q[:, 2])
    order = np.lexsort((np.arange(nv), key))
    G = (nv + LANES - 1) // LANES
    idx = np.empty(G * LANES, np.int64)
    idx[:nv] = order
    idx[nv:] = order[(G - 1) * LANES]
    gv = hv[idx].reshape(G, LANES, 3)
    c, r = _sphere(gv, gv.min(1), gv.max(1))
    bc, br = _sphere(hv, lo, hi)
    return gv, c, r, bc, br


def _perp2(c, o, d):
    cx, cy, cz = c[..., 0] - o[..., 0], c[..., 1] - o[..., 1], c[..., 2] - o[..., 2]
    dn2 = d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]
    t = cx * d[..., 0] + cy * d[..., 1] + cz * d[..., 2]
    return (cx * cx + cy * cy + cz * cz) - t * t / dn2, dn2


def near_far_groups(o, d, verts, geo_threshold, slack=(1.01, 1e-5)):
    """k_near_far_groups with its culls applied per ray (the kernel culls the whole body per block of 64 rays, which can
    only test more groups): rays with a unit direction skip a group whose line distance from the group's centre exceeds
    (radius + threshold) * slack[0] + slack[1]; the same test against the whole mesh's sphere skips every group.
    `slack` other than the kernel's is for planting defects."""
    o, d = np.asarray(o, F32), np.asarray(d, F32)
    gv, gc, gr, bc, br = vertex_groups(verts)
    thr, _ = thr_sq(geo_threshold)
    m, a = F32(slack[0]), F32(slack[1])
    p_b, dn2 = _perp2(bc[None], o, d)
    unit = np.abs(dn2 - F32(1)) <= F32(1e-3)
    lim = (br + thr) * m + a
    body = ~unit | ~(p_b > lim * lim)
    near = np.full(o.shape[0], np.inf, F32)
    far = np.full(o.shape[0], -np.inf, F32)
    p_g, _ = _perp2(gc[None], o[:, None], d[:, None])                  # [R, G]
    lim_g = (gr + thr) * m + a
    test = body[:, None] & (~unit[:, None] | ~(p_g > lim_g * lim_g))
    for g in range(gv.shape[0]):
        rows = np.nonzero(test[:, g])[0]
        if len(rows):
            n, f = near_far_exhaustive(o[rows], d[rows], gv[g], geo_threshold)
            near[rows] = np.minimum(near[rows], n)
            far[rows] = np.maximum(far[rows], f)
    return near, far


def near_far_body_cull(o, d, verts, geo_threshold, slack=(1.001, 1e-6)):
    """k_near_far: the exhaustive loop behind its whole-body cull (k_vert_bounds' sphere, 0.1 % slack), per ray."""
    o, d, v = np.asarray(o, F32), np.asarray(d, F32), np.asarray(verts, F32)
    c, r = _sphere(v, v.min(0), v.max(0))
    thr, _ = thr_sq(geo_threshold)
    p, dn2 = _perp2(c[None], o, d)
    lim = (r + thr) * F32(slack[0]) + F32(slack[1])
    may = ~(p > lim * lim) | (np.abs(dn2 - F32(1)) > F32(1e-3))
    near = np.full(o.shape[0], np.inf, F32)
    far = np.full(o.shape[0], -np.inf, F32)
    if may.any():
        near[may], far[may] = near_far_exhaustive(o[may], d[may], v, geo_threshold)
    return near, far


# ---------------------------------------------------------------------------------------------
# cdf, inversion, importance sampling (build_cdf, invert_cdf, k_sample_pdf, k_importance)
# ---------------------------------------------------------------------------------------------
def _lanes(x, base):
    """columns base..base+31 of x [R, n] as [R, 32], zero-padded"""
    out = np.zeros((x.shape[0], LANES), x.dtype)
    blk = x[:, base:base + LANES]
    out[:, :blk.shape[1]] = blk
    return out


def build_cdf(w, drop_carry=False):
    """cdf [R, n+1] float32 from weights w [R, n]: lane partial sums of (w + 1e-5) in double, an xor-butterfly total
    rounded to float, then per 32-lane chunk a double Hillis-Steele scan of the float pdf plus the running carry, each
    prefix rounded to float.  drop_carry plants a defect (the chunks do not carry their predecessors' sum)."""
    w = np.asarray(w, F32)
    R, n = w.shape
    wp = w + F32(1e-5)
    part = np.zeros((R, LANES), F64)
    for base in range(0, n, LANES):
        part = part + _lanes(wp, base).astype(F64)
    lane = np.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        part = part + part[:, lane ^ o]
    total = part[:, :1].astype(F32)
    cdf = np.zeros((R, n + 1), F32)
    carry = np.zeros((R, 1), F64)
    for base in range(0, n, LANES):
        inc = _lanes(wp / total, base).astype(F64)
        for o in (1, 2, 4, 8, 16):
            nxt = inc.copy()
            nxt[:, o:] = inc[:, o:] + inc[:, :-o]
            inc = nxt
        k = min(LANES, n - base)
        cdf[:, base + 1:base + 1 + k] = (inc[:, :k] if drop_carry else carry + inc[:, :k]).astype(F32)
        carry = carry + inc[:, 31:32]
    return cdf


def searchsorted(cdf, u, right=True):
    """the kernel's binary search: number of entries <= u (right=True) or < u (right=False, a planted defect)"""
    R, B = cdf.shape
    lo = np.zeros(u.shape, np.int64)
    hi = np.full(u.shape, B, np.int64)
    rows = np.arange(R)[:, None]
    while True:
        act = lo < hi
        if not act.any():
            return lo
        mid = (lo + hi) >> 1
        c = cdf[rows, np.minimum(mid, B - 1)]
        go = (c <= u) if right else (c < u)
        lo = np.where(act & go, mid + 1, lo)
        hi = np.where(act & ~go, mid, hi)


def invert_cdf(cdf, bins, u, right=True, with_den=False):
    """invert_cdf for every u [R, N]: searchsorted, den < 1e-5 -> 1, linear interpolation between the bins."""
    B = cdf.shape[1]
    u = np.asarray(u, F32)
    lo = searchsorted(cdf, u, right)
    below, above = np.maximum(0, lo - 1), np.minimum(B - 1, lo)
    rows = np.arange(cdf.shape[0])[:, None]
    c0, c1 = cdf[rows, below], cdf[rows, above]
    b0, b1 = bins[rows, below], bins[rows, above]
    den = c1 - c0
    out = b0 + (u - c0) / np.where(den < F32(1e-5), F32(1), den) * (b1 - b0)
    return (out.astype(F32), den) if with_den else out.astype(F32)


def sample_pdf(bins, weights, N, u=None, **defect):
    bins = np.asarray(bins, F32)
    if u is None:
        u = np.broadcast_to(linspace01(np.arange(N), N), (bins.shape[0], N))
    cdf = build_cdf(weights, drop_carry=defect.get("drop_carry", False))
    return invert_cdf(cdf, bins, u, right=defect.get("right", True))


def importance(o, d, z, w, N, including_old=True, **defect):
    """k_importance: (pts [R,T,3], z [R,T]) with the inverse-cdf samples on the bin mids of z and the cdf of
    w[:, 1:-1]; with including_old the union with z, sorted."""
    z = np.asarray(z, F32)
    mids = F32(0.5) * (z[:, 1:] + z[:, :-1])
    zn = sample_pdf(mids, np.asarray(w, F32)[:, 1:-1], N, **defect)
    zo = np.sort(np.concatenate([z, zn], 1), 1, kind="stable") if including_old else zn
    o, d = np.asarray(o, F32), np.asarray(d, F32)
    return o[:, None, :] + d[:, None, :] * zo[..., None], zo


def merge(z_list, raw_list=None, stable=True):
    """k_merge: the (z, position in the concatenated list) order -- a stable sort by z; stable=False plants a defect
    (ties broken the other way)."""
    zc = np.concatenate([np.asarray(z, F32) for z in z_list], 1)
    pos = np.broadcast_to(np.arange(zc.shape[1]), zc.shape)
    order = np.lexsort((pos if stable else -pos, zc), axis=1) if zc.ndim == 2 else None
    zs = np.take_along_axis(zc, order, 1)
    if raw_list is None:
        return zs, None
    rc = np.concatenate([np.asarray(r, F32) for r in raw_list], 1)
    return zs, np.take_along_axis(rc, order[..., None], 1)


# ---------------------------------------------------------------------------------------------
# composite: float64 windows (k_raw2outputs, k_raw2outputs_bwd)
# ---------------------------------------------------------------------------------------------
class Val:
    """An intermediate of an fp32 chain: f = float32 emulation, e = exact value (float64), B >= |kernel - e|."""
    __slots__ = ("f", "e", "B")

    def __init__(self, f, e=None, B=None):
        self.f = np.asarray(f, F32)
        self.e = self.f.astype(F64) if e is None else np.asarray(e, F64)
        self.B = np.zeros(self.e.shape) if B is None else np.asarray(B, F64)

    @staticmethod
    def _r(f, e, B):                           # one fp32 rounding of a result whose exact value is within B of e
        return Val(f, e, B + U * (np.abs(e) + B) + TINY)

    def __add__(a, b):
        b = _v(b)
        return Val._r(a.f + b.f, a.e + b.e, a.B + b.B)

    def __sub__(a, b):
        b = _v(b)
        return Val._r(a.f - b.f, a.e - b.e, a.B + b.B)

    def __radd__(a, b):
        return _v(b) + a

    def __rsub__(a, b):
        return _v(b) - a

    def __mul__(a, b):
        b = _v(b)
        return Val._r(a.f * b.f, a.e * b.e, np.abs(a.e) * b.B + np.abs(b.e) * a.B + a.B * b.B)

    def __truediv__(a, b):
        b = _v(b)
        q = a.e / b.e
        den = np.abs(b.e) - b.B
        with np.errstate(divide="ignore", invalid="ignore"):
            err = np.where(den > 0, (np.abs(q) * b.B + a.B) / den, np.inf)
        return Val._r(a.f / b.f, q, err)

    def __rtruediv__(a, b):
        return _v(b) / a

    def __getitem__(self, k):
        return Val(self.f[k], self.e[k], self.B[k])


def _v(x):
    return x if isinstance(x, Val) else Val(x)


def vexp(a):
    """expf: at most 2 ulp (<= 2^-22 |result|) from exp of the computed argument"""
    y = np.exp(a.e)
    err = y * np.expm1(a.B)
    return Val(np.exp(a.f), y, err + 2.0 ** -22 * (y + err) + TINY)


def vsel(mask, a, b):
    a, b = _v(a), _v(b)
    return Val(np.where(mask, a.f, b.f), np.where(mask, a.e, b.e), np.where(mask, a.B, b.B))


def vcat(vals, axis=1):
    return Val(np.concatenate([v.f for v in vals], axis), np.concatenate([v.e for v in vals], axis),
               np.concatenate([v.B for v in vals], axis))


def _shift_up(v, o, fill):
    """__shfl_up_sync(v, o) with lanes < o taking `fill`"""
    f = np.full(v.f.shape, fill, F32)
    e = np.full(v.e.shape, float(fill))
    B = np.zeros(v.B.shape)
    f[:, o:], e[:, o:], B[:, o:] = v.f[:, :-o], v.e[:, :-o], v.B[:, :-o]
    return Val(f, e, B)


def _shift_down(v, o, fill):
    f = np.full(v.f.shape, fill, F32)
    e = np.full(v.e.shape, float(fill))
    B = np.zeros(v.B.shape)
    f[:, :-o], e[:, :-o], B[:, :-o] = v.f[:, o:], v.e[:, o:], v.B[:, o:]
    return Val(f, e, B)


def _butterfly(v):
    lane = np.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, lane ^ o]
    return v[:, 0]


def _prefix(raw, z, d, noise, sigma_scale):
    """the exactly restated fp32 prefix of both kernels: dnorm, dist, sigma and the exp argument (all correctly
    rounded), padded to whole 32-lane chunks"""
    raw, z, d = np.asarray(raw, F32), np.asarray(z, F32), np.asarray(d, F32)
    R, S = z.shape
    dnorm = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])[:, None]
    dist = np.concatenate([z[:, 1:] - z[:, :-1], np.full((R, 1), 1e10, F32)], 1) * dnorm
    sg = raw[..., 3] * F32(sigma_scale)
    if noise is not None:
        sg = sg + np.asarray(noise, F32)
    x = -np.maximum(sg, F32(0)) * dist
    P = -(-S // LANES) * LANES
    pad = lambda a, v: np.concatenate([a, np.full((R, P - S), v, a.dtype)], 1)
    return dict(R=R, S=S, P=P, live=pad(np.ones((R, S), bool), False), z=pad(z, 0), dist=pad(dist, 0), sg=pad(sg, 0),
                x=pad(x, 0), v=[pad(raw[..., c], 0) for c in range(3)])


def _alpha_f(p):
    """e = expf(x), alpha = 1 - e and f = 1 - alpha + 1e-10 per sample.  alpha and f are the fp32 values computed from
    the correctly rounded exp (the exact chain starts from them); their bound covers the kernel's expf being up to 2 ulp
    away, by evaluating the same fp32 steps at e -+ 3 ulp (both steps are monotone in e).  This keeps the transmittance
    exact where 1 - e rounds to 1: f is then 1e-10 whichever e the kernel had, and Q / f stays well conditioned."""
    e = vexp(Val(p["x"]))
    e0 = np.exp(p["x"].astype(F64)).astype(F32)
    lo, hi = e0, e0
    for _ in range(3):
        lo, hi = np.nextafter(lo, F32(-1)), np.nextafter(hi, F32(2))
    lo = np.maximum(lo, F32(0))

    def af(ev):
        a = F32(1) - ev
        return a, (F32(1) - a) + F32(1e-10)
    (a0, f0), (a1, f1), (a2, f2) = af(e0), af(lo), af(hi)
    spread = lambda v0, v1, v2: np.maximum(np.abs(v1.astype(F64) - v0), np.abs(v2.astype(F64) - v0))
    alpha = vsel(p["live"], Val(a0, None, spread(a0, a1, a2)), 0.0)
    f = vsel(p["live"], Val(f0, None, spread(f0, f1, f2)), 1.0)
    return e, alpha, f


def _sigmoid(v):
    return 1.0 / (1.0 + vexp(Val(-v)))


def _trans(f, P):
    """exclusive transmittance: per chunk a Hillis-Steele product scan over the lanes, times the running carry"""
    T, incs = [], []
    carry = Val(np.ones((f.f.shape[0], 1), F32))
    lane = np.arange(LANES)
    for base in range(0, P, LANES):
        inc = f[:, base:base + LANES]
        for o in (1, 2, 4, 8, 16):
            inc = vsel(lane >= o, inc * _shift_up(inc, o, 1.0), inc)
        exc = _shift_up(inc, 1, 1.0)
        T.append(carry * exc)
        carry = carry * inc[:, 31:32]
    return vcat(T)


def composite_forward(raw, z, d, noise=None, sigma_scale=1.0, white_bkg=True):
    """k_raw2outputs as windows: dict of Val for w [R,S], rgb [R,3], acc, depth, disp [R]."""
    p = _prefix(raw, z, d, noise, sigma_scale)
    e, alpha, f = _alpha_f(p)
    T = _trans(f, p["P"])
    w = alpha * T
    c = [_sigmoid(p["v"][k]) for k in range(3)]
    zero = np.zeros((p["R"], LANES), F32)
    sums = {k: Val(zero) for k in ("r", "g", "b", "d", "a")}
    for base in range(0, p["P"], LANES):
        sl = slice(base, base + LANES)
        live = p["live"][:, sl]
        ws = w[:, sl]
        for k, term in (("r", ws * c[0][:, sl]), ("g", ws * c[1][:, sl]), ("b", ws * c[2][:, sl]),
                        ("d", ws * Val(p["z"][:, sl])), ("a", ws)):
            sums[k] = vsel(live, sums[k] + term, sums[k])
    s = {k: _butterfly(v) for k, v in sums.items()}
    rgb = [s["r"], s["g"], s["b"]]
    if white_bkg:
        bgw = 1.0 - s["a"]
        rgb = [x + bgw for x in rgb]
    q = s["d"] / s["a"]
    ok = (q.e - q.B > 1e-10) & np.isfinite(q.B)                 # max(1e-10, q) is q over the whole window
    disp = 1.0 / q
    disp = Val(disp.f, disp.e, np.where(ok, disp.B, np.inf))
    S = p["S"]
    return dict(w=w[:, :S], rgb=Val(np.stack([x.f for x in rgb], 1), np.stack([x.e for x in rgb], 1),
                                    np.stack([x.B for x in rgb], 1)),
                acc=s["a"], depth=s["d"], disp=disp)


def composite_backward(raw, z, d, g_rgb=None, g_depth=None, g_acc=None, g_w=None, noise=None, sigma_scale=1.0,
                       white_bkg=True, suffix="shift"):
    """k_raw2outputs_bwd as windows: Val [R,S,4] of d raw.  suffix = "shift" is the kernel's exclusive suffix (the next
    lane's inclusive sum); "subtract" plants the cancelling inc - G*w form."""
    p = _prefix(raw, z, d, noise, sigma_scale)
    R, S, P = p["R"], p["S"], p["P"]
    zr = np.zeros(R, F32)
    gr, gg, gb = ((np.asarray(g_rgb, F32)[:, k] if g_rgb is not None else zr)[:, None] for k in range(3))
    gd = (np.asarray(g_depth, F32) if g_depth is not None else zr)[:, None]
    ga = (np.asarray(g_acc, F32) if g_acc is not None else zr)[:, None]
    gw = np.zeros((R, P), F32)
    if g_w is not None:
        gw[:, :S] = np.asarray(g_w, F32)
    wsub = (gr + gg + gb) if white_bkg else np.zeros((R, 1), F32)
    e, alpha, f = _alpha_f(p)
    T = _trans(f, p["P"])
    w = alpha * T
    c = [_sigmoid(p["v"][k]) for k in range(3)]
    G = Val(gr) * c[0] + Val(gg) * c[1] + Val(gb) * c[2] - Val(wsub) + Val(gd) * Val(p["z"]) + Val(ga) + Val(gw)
    Gw = vsel(p["live"], G * w, 0.0)
    GT = G * T
    d_rgb = [Val(g) * w * c[k] * (1.0 - c[k]) for k, g in enumerate((gr, gg, gb))]
    lane = np.arange(LANES)
    tail = Val(np.zeros((R, 1), F32))
    Q = [None] * (P // LANES)
    for base in range(P - LANES, -1, -LANES):
        x = Gw[:, base:base + LANES]
        inc = x
        for o in (1, 2, 4, 8, 16):
            inc = vsel(lane + o < LANES, inc + _shift_down(inc, o, 0.0), inc)
        if suffix == "shift":
            Q[base // LANES] = tail + _shift_down(inc, 1, 0.0)
        else:
            Q[base // LANES] = tail + (inc - x)
        tail = tail + inc[:, 0:1]
    Q = vcat(Q)
    dalpha = GT - Q / f
    dsig = dalpha * Val(p["dist"]) * e * F32(sigma_scale)
    dsig = vsel(p["sg"] > 0, dsig, 0.0)
    out = [x[:, :S] for x in d_rgb + [dsig]]
    return Val(np.stack([x.f for x in out], -1), np.stack([x.e for x in out], -1), np.stack([x.B for x in out], -1))


# ---------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------
def first_diff(name, got, want):
    """None if got and want are bitwise the same values (NaN == NaN), else a description of the first differing element"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    if same.all():
        return None
    i = tuple(int(k) for k in np.argwhere(~same)[0])
    return f"{name}: {int((~same).sum())} of {same.size} differ; first at {i}: got {got[i]!r}, want {want[i]!r}"


def outside(name, got, v):
    """None if every element of got lies in [v.e - v.B, v.e + v.B], else the first element outside, with its window"""
    got = np.asarray(got, F64)
    ok = (np.abs(got - v.e) <= v.B) | np.isposinf(v.B)             # an infinite bound: no claim (disp at acc ~ 0)
    if ok.all():
        return None
    i = tuple(int(k) for k in np.argwhere(~ok)[0])
    rel = abs(got[i] - v.e[i]) / max(abs(v.e[i]), 1e-300)
    return (f"{name}: {int((~ok).sum())} of {ok.size} outside the window; first at {i}: got {got[i]!r}, "
            f"exact {v.e[i]!r}, bound {v.B[i]!r} (relative error {rel:.3g})")
