"""Exact windows for the weight and bias gradients of the tensor-core training step: k_dw_gemm (csrc/dw_gemm.cu), the
narrow cuBLAS GEMMs and fp32 sums of neuman_b200.autograd._weight_grads, and their assembly into the gradient of every
nn.Linear of NeRF.forward (models/vanilla.py:120-152).

Every gradient element is a sum over the n samples of g * x: g from an fp16 gradient plane (the loss scale S = 1/inv
included), x from an fp16 activation or encoding plane, or 1 for a bias.  Products of fp16 values are exact in float64,
so e = the float64 sum (exact up to float64 rounding), and B bounds what an fp32 evaluation in the code's order adds:
    k_dw_gemm             dw_window              any contiguous 64-row split into CTAs, K = 16 MMAs, red.add across CTAs
    cuBLAS torch.mm       gemm_window_any_order  any summation order (no assumption on cuBLAS's kernel or split-K)
    fp32 torch sum        sum_window             any summation order
An fp32 gradient v is correct when |v - e| <= B on every element.  The windows are per element, never scaled by a
matrix norm, so an element whose exact value is small next to its matrix is held to its own size.  Multiplying by inv
(a power of two) is exact.  Works on CPU and CUDA tensors; no GPU needed."""
import torch

from tests import tc_exact as tx

EPS32 = tx.EPS32                      # 2^-23: fp32 truncation (2u for round-to-nearest)
U32 = 2.0 ** -24                      # fp32 round-to-nearest unit roundoff
GAMMA16 = 16.001 * EPS32              # one K = 16 wgmma (tc_exact.mma_ref)
FLUSH = 2.0 ** -126                   # what one flush of an fp32 subnormal to zero can lose
MIN16 = 2.0 ** -14                    # smallest normal fp16
DW_ROWS = 64                          # csrc/dw_gemm.cu: K rows per pipeline stage, the granularity of the CTA split
DW_MAX_WORK = 74                      # csrc/dw_gemm.cu: most work items (CTA pairs) of one launch
DW_STAGES = 4                         # csrc/dw_gemm.cu: slots of the stage ring
CHUNK_ROWS = 16 * 512                 # rows per float64 block of the prefix-range pass


def n_parts_max(n):
    """The most CTAs that can add a partial into one output element: one per 64-row range, at most DW_MAX_WORK."""
    return max(1, min(-(-n // DW_ROWS), DW_MAX_WORK))


def _ones(n, like):
    return torch.ones(n, 1, dtype=torch.float64, device=like.device)


def mma_abs(t):
    """|t| as the tensor cores (k_dw_gemm's wgmma, cuBLAS) align it: an fp16 subnormal operand counts as the smallest normal, 2^-14.  Measured on
    the H100 (DESIGN.md §2; pinned by tests/test_gpu_dw_exact.py::test_subnormal_operands): products of subnormal
    operands are aligned by that exponent, not by their own, so their rounding error is relative to 2^-14 |x|, up to
    2^10 times |g x|.  Operands of normal size are unaffected."""
    a = t.abs()
    return torch.where((a > 0) & (a < MIN16), torch.full_like(a, MIN16), a)


def prefix_stats(G, X, chunk_rows=CHUNK_ROWS, align_subnormals=True):
    """D = G^T X over the rows (G [n, M], X [n, N], X = None for a column of ones) in float64 ->
    (e [M, N], S = sum mma_abs(g) mma_abs(x), R = max_j P_j - min_j P_j) with P_j = the sum over rows < 16 j,
    j = 0 .. ceil(n/16): the
    prefix sums at the granularity of one MMA.  Computed 16 rows at a time by batched GEMMs, chunk by chunk, carrying the
    running prefix, minimum and maximum, so no [n/16, M, N] tensor is ever held."""
    n, M = G.shape
    N = 1 if X is None else X.shape[1]
    run = torch.zeros(M, N, dtype=torch.float64, device=G.device)
    lo, hi, S = run.clone(), run.clone(), run.clone()     # P_0 = 0 is a prefix too
    for r0 in range(0, n, chunk_rows):
        r1 = min(n, r0 + chunk_rows)
        g = G[r0:r1].double()
        x = _ones(r1 - r0, g) if X is None else X[r0:r1].double()
        S += (mma_abs(g).T @ mma_abs(x)) if align_subnormals else (g.abs().T @ x.abs())
        pad = -(r1 - r0) % 16                               # rows past n: zeros, as TMA fills them
        if pad:
            g = torch.cat([g, g.new_zeros(pad, M)])
            x = torch.cat([x, x.new_zeros(pad, N)])
        k = g.shape[0] // 16
        P = torch.bmm(g.reshape(k, 16, M).transpose(1, 2), x.reshape(k, 16, N))    # [k, M, N] one MMA each
        P = P.cumsum_(0).add_(run)
        lo = torch.minimum(lo, P.amin(0))
        hi = torch.maximum(hi, P.amax(0))
        run = P[-1].clone()
        del P
    return run, S, hi - lo


def dw_window(G, X, n_parts=None, align_subnormals=True):
    """(e, B) of k_dw_gemm's D = G^T X (K = n; X = None: the bias gradient, X = 1).  How the kernel sums:
    a work item's rows are split into contiguous 64-row ranges, one per CTA; a CTA consumes its range in ascending order
    as K = 16 wgmma instructions into fp32 registers; the CTAs' partials are red.global.add-ed into a zeroed output in any
    order.  The bound holds for ANY such split into at most n_parts ranges (default: n_parts_max(n)), so it does not
    restate the host's SM-count-dependent work list.
      MMA term: instruction j adds at most GAMMA16 (|acc| + B_acc + S_j) (tc_exact.mma_ref; S_j with mma_abs, which
        only matters for fp16 subnormal operands).  A CTA's running partial
        is P_r - P_r0, so |acc| <= R = max P - min P; summed over the m = ceil(n/16) instructions of all CTAs,
        B_mma = GAMMA16 (m R + S) / (1 - GAMMA16 m).
      Reduction term: p partials, each at most R + B_mma in size, added by p - 1 rounding fp32 adds (the first lands on
        0 exactly): gamma_{p-1} p (R + B_mma), u = 2^-24.
      Flush term: red.add.f32 and atomicAdd(float) flush subnormals: p 2^-126.
    align_subnormals=False gives the window without the subnormal allowance of mma_abs."""
    n = G.shape[0]
    e, S, R = prefix_stats(G, X, align_subnormals=align_subnormals)
    m = -(-n // 16)
    p = n_parts_max(n) if n_parts is None else int(n_parts)
    Bm = GAMMA16 * (m * R + S) / (1.0 - GAMMA16 * m)
    g_red = (p - 1) * U32 / (1.0 - (p - 1) * U32)
    B = Bm + g_red * p * (R + Bm) + p * FLUSH
    return e, B


def gemm_window_any_order(G, X, chunk_rows=CHUNK_ROWS, align_subnormals=True):
    """(e, B) of neuman_b200.autograd._wgrad: cuBLAS GEMMs G^T X with fp16 operands and fp32 output over fixed row
    blocks, their fp32 sum (K = n; X = None: a column of ones).  cuBLAS's kernel choice and order are unknown, so the
    bound is order-free.  It assumes that every addition on
    the way from the n exact products to the fp32 result is an fp32 (or wider) addition that rounds once, to nearest or
    toward zero, or a K = 16 MMA that adds at most GAMMA16 of its |accumulator| + |products| -- including the reduction of
    split-K partials.  Then each product passes at most k = n + 16 (the MMA chain) + ceil(n/16) (a split-K reduction of up
    to one partial per 16 rows) rounding steps: B = gamma_k S with u = 2^-23, plus ceil(n/16) flushes of a subnormal.
    A reduction below fp32 lies outside it: one cuBLAS GEMM with K = n picks such a split for some shapes, which is why
    _wgrad splits K itself.  S with mma_abs: cuBLAS runs on the same tensor cores, and its subnormal channels need the
    allowance too (test_subnormal_operands); align_subnormals=False gives the window without it."""
    n, M = G.shape
    N = 1 if X is None else X.shape[1]
    e = torch.zeros(M, N, dtype=torch.float64, device=G.device)
    S = e.clone()
    for r0 in range(0, n, chunk_rows):
        g = G[r0:r0 + chunk_rows].double()
        x = _ones(g.shape[0], g) if X is None else X[r0:r0 + chunk_rows].double()
        e += g.T @ x
        S += (mma_abs(g).T @ mma_abs(x)) if align_subnormals else (g.abs().T @ x.abs())
    k = n + 16 + -(-n // 16)
    return e, k * EPS32 / (1.0 - k * EPS32) * S + -(-n // 16) * FLUSH


def sum_window(g):
    """(e, B) of torch's fp32 g.sum(0) (g [n, c] fp32; the head biases): any order, n - 1 rounding adds,
    B = gamma_n sum |g| with u = 2^-24."""
    g = g.double()
    n = g.shape[0]
    return g.sum(0), n * U32 / (1.0 - n * U32) * g.abs().sum(0)


# ---------------------------------------------------------------------------------------------
# The layout of every parameter gradient, written from the reference's module (models/vanilla.py:120-152): which tensor
# each nn.Linear reads, in which column order; and which engine of _weight_grads sums which block
# ---------------------------------------------------------------------------------------------
KINDS = {                             # kind -> (position-encoding width, direction-encoding width or None)
    "posenc": (63, 27), "rotate": (63, 27),
    "carrier": (63, 27),              # the OffsetNet's Joiner carrier (models.offset_joiner_weights, DESIGN.md §7b)
    "nerft": (84, 27),                # position input (x, y, z, t): 4 + 2 * 4 * 10 channels in the reference's order
    "viewless": (63, None),           # use_viewdirs=False: output_linear reads h7
}


def layout(viewless):
    """[(nn.Linear, gradient of its output, [(input block, engine), ...] in the module's column order, bias engine)].
    Inputs: pe / dpe = Embedder outputs of the position / direction, sx{l} = h after pts_linears.l (ReLU'd), sf = feature,
    sv = h after views_linears.0.  Gradients: g_pre{l}, g_f, g_v = dL/d(pre-activation) times the loss scale; g8 = the
    fp16 operand r16(S dL/d raw) of the heads.  Engines: dw = k_dw_gemm, mm = cuBLAS, sum = fp32 torch sum of dL/d raw."""
    L = [("pts_linears.0", "g_pre0", [("pe", "mm")], "mm")]              # the bias: the constant-1 column of the plane
    for l in range(1, 8):
        ins = [("pe", "mm"), ("sx4", "dw")] if l == 5 else [(f"sx{l - 1}", "dw")]   # skip: cat([input_pts, h]) (:131)
        L.append((f"pts_linears.{l}", f"g_pre{l}", ins, "dw"))
    if viewless:
        L.append(("output_linear", "g8", [("sx7", "mm")], "sum"))                   # :146
    else:
        L += [("alpha_linear", "g8_alpha", [("sx7", "mm")], "sum"),                 # :136, reads h7 like feature_linear
              ("feature_linear", "g_f", [("sx7", "dw")], "dw"),                     # :137
              ("views_linears.0", "g_v", [("sf", "dw"), ("dpe", "mm")], "dw"),      # :138 cat([feature, input_views])
              ("rgb_linear", "g8_rgb", [("sv", "mm")], "sum")]                      # :144
    return L


HEAD_COLS = {"g8": slice(0, 4), "g8_alpha": slice(3, 4), "g8_rgb": slice(0, 3)}


def param_windows(kind, planes, inv, n_parts=None):
    """{parameter name: (e, B)} for every parameter of a Joiner of `kind` (KINDS), from the planes one training step
    used: g (dL/d raw [n,4] fp32), g_pre [8,n,256], g_f, g_v (fp16, times the loss scale 1/inv), sx [8,n,256], sf, sv
    (the forward's stash), pe / dpe (the encodings as the forward multiplied them; only their first KINDS[kind] columns
    are read).  e is built from the fp16 operands the code multiplies, r16(g S) for the heads included."""
    n_pe, n_dpe = KINDS[kind]
    viewless = n_dpe is None
    inv = float(inv)
    g32 = planes['g']
    g8 = tx.r16(g32.double() / inv)
    ins = {f"sx{l}": planes['sx'][l] for l in range(8)}
    ins['pe'] = planes['pe'][:, :n_pe]
    grads = {f"g_pre{l}": planes['g_pre'][l] for l in range(8)}
    grads.update({k: g8[:, c] for k, c in HEAD_COLS.items()})
    if not viewless:
        ins.update(sf=planes['sf'], sv=planes['sv'], dpe=planes['dpe'][:, :n_dpe])
        grads.update(g_f=planes['g_f'], g_v=planes['g_v'])
    engines = {"dw": lambda G, X: dw_window(G, X, n_parts), "mm": gemm_window_any_order}
    out = {}
    for name, gk, blocks, bias_engine in layout(viewless):
        G = grads[gk]
        es, Bs = [], []
        for x, engine in blocks:
            e, B = engines[engine](G, ins[x])
            es.append(e * inv)
            Bs.append(B * abs(inv))
        out[name + ".weight"] = (torch.cat(es, 1), torch.cat(Bs, 1))
        if bias_engine == "sum":
            out[name + ".bias"] = sum_window(g32[:, HEAD_COLS[gk]])
        else:
            e, B = engines[bias_engine](G, None)
            out[name + ".bias"] = (e[:, 0] * inv, B[:, 0] * abs(inv))
    return out


# ---------------------------------------------------------------------------------------------
# Gradient and activation planes for k_dw_gemm: plain ones, and adversarial ones
# ---------------------------------------------------------------------------------------------
def dw_planes(n, seed, device, width=256, views=128, adversarial=True):
    """The five input planes of nm_dw_gemm as fp16: g_pre [8,n,width], g_f [n,width], g_v [n,views], sx [8,n,width],
    sf [n,width].  Plain: ReLU-sparse activations, gradients masked on half of their entries.  Adversarial, on top:
    row kinds mixed at random -- rows of +-60000 next to rows of 1e-3, gradient rows in the fp16 subnormal range, all-zero
    rows -- exactly cancelling row pairs (row i + 1 = -row i in every gradient plane, the same activation row: e gets 0
    from them and S a lot), and whole gradient channels at subnormal and at 1e-3 scale, so that some elements see nothing
    else."""
    gen = torch.Generator(device=device).manual_seed(seed)

    def rnd(*s):
        return torch.randn(*s, generator=gen, device=device)

    def uni(*s):
        return torch.rand(*s, generator=gen, device=device)

    def grad(*s):
        return rnd(*s) * 0.5 * (uni(*s) < 0.5)

    def act(*s, signed=False):
        x = rnd(*s) * 1.5
        return x if signed else torch.relu(x)

    G = [grad(8, n, width), grad(n, width), grad(n, views)]
    X = [act(8, n, width), act(n, width, signed=True)]
    if adversarial:
        kind = torch.randint(0, 8, (n,), generator=gen, device=device)
        rows = {k: (kind == k).view(n, 1) for k in range(4, 8)}
        for i, t0 in enumerate(G):
            big = torch.sign(rnd(*t0.shape)) * 60000.0 * (uni(*t0.shape) < 0.25)
            t = torch.where(rows[4], big + t0, t0)                                   # +-60000 on a quarter of the channels
            t = torch.where(rows[5], t * 1e-3, t)
            t = torch.where(rows[6], t * 2.0 ** -18, t)                              # fp16 subnormals: multiples of 2^-24
            t = torch.where(rows[7], torch.zeros_like(t), t)
            t[..., :4] = t0[..., :4] * 2.0 ** -18                                    # subnormal channels
            t[..., 4:8] = t0[..., 4:8] * 1e-3
            G[i] = t
        for i, t in enumerate(X):
            t = torch.where(rows[4], t.abs().clamp_min(0.5) * 2.0e4 * torch.sign(t), t)
            t = torch.where(rows[5], t * 1e-3, t)
            t = torch.where(rows[7] & (uni(n, 1) < 0.5), torch.zeros_like(t), t)
            X[i] = t
        pair = torch.nonzero(uni(n // 2) < 0.15).view(-1) * 2                         # rows (i, i + 1), i even
        pair = pair[pair + 1 < n]
        for t in G:
            t[..., pair + 1, :] = -t[..., pair, :]
        for t in X:
            t[..., pair + 1, :] = t[..., pair, :]
    g_pre, g_f, g_v = (t.clamp(-60000, 60000).half() for t in G)
    sx, sf = (t.clamp(-60000, 60000).half() for t in X)
    return dict(g_pre=g_pre, g_f=g_f, g_v=g_v, sx=sx, sf=sf)


def dw_items(planes, trunk_only=False):
    """The work items of nm_dw_gemm as (G, X) pairs in output order: item k < 7 = pts_linears k+1 (g_pre[k+1], sx[k]),
    7 = feature_linear (g_f, sx[7]), 8 = views_linears.0's feature columns (g_v, sf)."""
    p = planes
    items = [(p['g_pre'][k + 1], p['sx'][k]) for k in range(7)]
    if not trunk_only:
        items += [(p['g_f'], p['sx'][7]), (p['g_v'], p['sf'])]
    return items


def used(v, e, B):
    """max |v - e| / B (0/0 = 0): how much of its proven window the result takes"""
    d = (v.double() - e).abs()
    r = torch.where(d > 0, d / B.clamp_min(1e-300), torch.zeros_like(d))
    return float(r.max()) if r.numel() else 0.0


def assert_in_window(name, v, e, B):
    c = tx.check32(name, v, e, B)
    assert c.ok.all(), c.message()
    return c
