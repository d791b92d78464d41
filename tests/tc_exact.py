"""Exact windows for the tensor-core MLP (csrc/mlp_tc.cu, csrc/mlp_tc_bwd.cu): every output element of a layer is a
correct fp32 accumulation of fp16 operands, then (for fp16 outputs) a round-to-nearest to fp16.

For an output y = sum_k a_k b_k (+ bias) the operands a, b are the exact fp16 values the kernel consumed (its own stash
planes and encodings, the fp16-rounded weights).  Products of fp16 values are exact in float64, so
    e = the sum in float64                                  (exact up to float64 rounding)
    B = a bound on the error of the fp32 accumulation      (mma_ref: in the order the kernel issues its K = 16 MMAs)
B holds for fp32 adders that round to nearest or truncate.  Then
    fp16 outputs:  r16(f(e - B)) <= v <= r16(f(e + B))     f = ReLU, a 0/1 mask or the identity
    fp32 outputs:  |v - e| <= B (+ the rounding of a final fp32 add)
Rounding is monotone, so this is an all-elements check; an element may differ from r16(e) only when e lies within B of
a rounding midpoint.  Each layer is checked on the kernel's own inputs, so an error does not propagate and a failure
names one layer, row and column.  Works on CPU and CUDA tensors; no GPU needed."""
import math

import torch

EPS32 = 2.0 ** -23          # fp32 unit roundoff for truncation (2u for round-to-nearest)


def r16(x):
    """Round float64 to the nearest fp16 (through fp32: for an fp32 accumulator v >= x, r16 of the fp32 rounding of x
    is still <= r16(v), so the window stays a proof).  Beyond the fp16 range this is +-inf."""
    return x.float().half().double()


def affine(a, W, b=None):
    """e = a @ W^T (+ b) and S = |a| @ |W|^T (+ |b|) in float64."""
    a, W = a.double(), W.double()
    e, S = a @ W.T, a.abs() @ W.abs().T
    if b is not None:
        b = b.double()
        e, S = e + b, S + b.abs()
    return e, S


def mma_ref(blocks):
    """(e, B) of a wgmma accumulation: `blocks` = [(a [n, k], W [N, k]), ...] in the kernel's K order, consumed 16
    channels per instruction.  Each instruction computes D = A B + D (PTX: in issue order); inside one instruction the
    16 exact products and the accumulator are summed in fp32 in ANY order, so instruction j adds at most
    16 * 2^-23 * (|E_{j-1}| + B_{j-1} + S_j) to the error, E_{j-1} being the exact partial sum before it and S_j the sum of
    |products| of its 16 channels.  B is the sum of those terms: a proof for truncating or rounding fp32 adders, ~K/16
    times tighter than the order-free bound K 2^-23 sum|a_k b_k|."""
    e = B = None
    g = 16.001 * EPS32                                     # gamma_16 = 16u / (1 - 16u), rounded up
    for a, W in blocks:
        a, W = a.double(), W.double()
        for k0 in range(0, a.shape[1], 16):
            aj, Wj = a[:, k0:k0 + 16], W[:, k0:k0 + 16]
            p, s = aj @ Wj.T, aj.abs() @ Wj.abs().T
            if e is None:
                e, B = p, g * s
            else:
                B = B + g * (e.abs() + B + s)
                e = e + p
    return e, B


class Check:
    """Result of one output plane against its window: `ok` per element, the window [lo, hi] and the diagnostics."""

    def __init__(self, name, v, lo, hi, e, B):
        self.name, self.v, self.lo, self.hi, self.e, self.B = name, v, lo, hi, e, B
        # NaN windows (an inf - inf in the reference) accept nothing; inf windows accept only the matching inf
        self.ok = (v >= lo) & (v <= hi)

    @property
    def n_bad(self):
        return int((~self.ok).sum())

    @property
    def occupancy(self):
        """fraction of elements whose window holds more than one representable value"""
        return float((self.lo != self.hi).double().mean()) if self.lo.numel() else 0.0

    def first_bad(self):
        idx = (~self.ok).nonzero()
        if not len(idx):
            return None
        i = tuple(int(t) for t in idx[0])
        return dict(layer=self.name, index=i, got=float(self.v[i]), expect=float(self.e[i]), B=float(self.B[i]),
                    lo=float(self.lo[i]), hi=float(self.hi[i]))

    def message(self):
        return f"{self.name}: {self.n_bad} of {self.ok.numel()} elements outside the window; first {self.first_bad()}"


def check16(name, v, e, B, relu=False, mask=None):
    """fp16 output v against r16(f(e -+ B)); f = ReLU and/or a 0/1 mask (masked elements must be exactly 0)."""
    lo, hi = e - B, e + B
    if relu:
        lo, hi = lo.clamp_min(0.0), hi.clamp_min(0.0)
    if mask is not None:
        lo, hi = torch.where(mask, lo, torch.zeros_like(lo)), torch.where(mask, hi, torch.zeros_like(hi))
    return Check(name, v.double(), r16(lo), r16(hi), e, B)


def check32(name, v, e, B):
    """fp32 output v against |v - e| <= B."""
    v = v.double()
    return Check(name, v, e - B, e + B, e, B)


def fma_chain_bound(parts, tail):
    """Error bound of an fp32 FMA chain acc = fma(x_i, w_i, acc) over the columns of `parts` [n, m] = x_i w_i (exact),
    left to right from 0: every step rounds once (<= 2^-23 |partial|); part i carries its own error bound tail[:, i]."""
    P, Bt = torch.cumsum(parts, 1), torch.cumsum(tail, 1)
    return Bt[:, -1] + EPS32 * (P.abs() + Bt).sum(1)


# ---------------------------------------------------------------------------------------------
# Layer-local references of the forward, in the kernel's K order (csrc/mlp_tc.cu; DESIGN.md §3/§4: the hidden biases
# are fp16 operands that ride in the MMAs, the alpha head is fp32 on the unrounded layer-7 accumulators, the rgb / alpha
# biases are fp32 adds)
# ---------------------------------------------------------------------------------------------
def weights(joiner, device):
    """(W16, W32): the network's parameters rounded to fp16 (what the packed slabs hold) and as fp32, both in float64."""
    sd = {k: v.detach().to(device) for k, v in joiner.nerf.state_dict().items()}
    return {k: v.half().double() for k, v in sd.items()}, {k: v.double() for k, v in sd.items()}


def n_pos(W16):
    return W16['pts_linears.0.weight'].shape[1]          # 63


def _bias_slab(pe, b):
    """The K = 16 bias MMA of a K = 256 step: channels 48..63 of the position encoding against a slab that is zero
    except for the column of channel 63 (= 1), which holds the bias."""
    W = torch.zeros(b.shape[0], 16, dtype=torch.float64, device=b.device)
    W[:, 15] = b
    return pe[:, 48:64], W


def hidden_blocks(W16, l, pe, sx, bias=True):
    """The (operand, weight) blocks of pts_linears.l in the order k_mlp_tc issues them (pe [n,64] with channel 63 = 1)."""
    w, b = W16[f'pts_linears.{l}.weight'], W16[f'pts_linears.{l}.bias']
    npe = n_pos(W16)
    if l in (0, 5):                                          # position-encoding block first, the bias in its column 63
        pe_w = torch.cat([w[:, :npe], b[:, None] if bias else 0 * b[:, None]], 1)
        return [(pe, pe_w)] + ([(sx[4], w[:, npe:])] if l == 5 else [])
    return [(sx[l - 1], w)] + ([_bias_slab(pe, b)] if bias else [])


def forward_checks(W16, W32, pe, dpe, sx, sf, sv, raw):
    """Yields a Check for every output of the training forward: layers 0..7, feature, views, rgb, alpha.
    pe [n,64] / dpe [n,32]: the fp16 encodings (nm_encode_f16); sx [8,n,256], sf, sv, raw: the kernel's outputs."""
    e7 = B7 = None
    for l in range(8):
        e, B = mma_ref(hidden_blocks(W16, l, pe, sx))
        if l == 7:
            e7, B7 = e, B
        yield check16(f"layer{l}", sx[l], e, B, relu=True)
    e, B = mma_ref([(sx[7], W16['feature_linear.weight']), _bias_slab(pe, W16['feature_linear.bias'])])
    yield check16("feature", sf, e, B)
    wv, ndpe = W16['views_linears.0.weight'], dpe.shape[1]
    dir_w = torch.zeros(wv.shape[0], ndpe, dtype=torch.float64, device=wv.device)
    dir_w[:, :wv.shape[1] - 256] = wv[:, 256:]
    dir_w[:, wv.shape[1] - 256] = W16['views_linears.0.bias']          # the bias column meets the constant channel
    e, B = mma_ref([(sf, wv[:, :256]), (dpe, dir_w)])
    yield check16("views", sv, e, B, relu=True)
    # rgb: the fp32 accumulator of sv @ W16_rgb^T (K = 128), then one fp32 add of the fp32 bias
    e, B = mma_ref([(sv, W16['rgb_linear.weight'])])
    e = e + W32['rgb_linear.bias']
    yield check32("rgb", raw[:, :3], e, B + EPS32 * (e.abs() + B))
    # alpha: each of the 4 threads of a row runs an fp32 FFMA chain over its 64 columns c = 8j + 2q + {1, 0} on
    # relu(acc7) with fp32 weights; two shuffle adds (pairs, then the halves) and the fp32 bias add follow.
    # |relu(acc7) - relu(e7)| <= B7 enters through |w_alpha|.
    wa, ba = W32['alpha_linear.weight'][0], W32['alpha_linear.bias']
    r = e7.clamp_min(0.0)
    t = r * wa
    tb = B7 * wa.abs()
    chains, cb = [], []
    for q in range(4):
        cols = torch.tensor([8 * j + 2 * q + o for j in range(32) for o in (1, 0)], device=r.device)
        chains.append(t[:, cols].sum(1))
        cb.append(fma_chain_bound(t[:, cols], tb[:, cols]))
    pair = [chains[0] + chains[1], chains[2] + chains[3]]
    pb = [cb[0] + cb[1] + EPS32 * (pair[0].abs() + cb[0] + cb[1]), cb[2] + cb[3] + EPS32 * (pair[1].abs() + cb[2] + cb[3])]
    tot = pair[0] + pair[1]
    Bt = pb[0] + pb[1] + EPS32 * (tot.abs() + pb[0] + pb[1])
    ea = tot + ba
    yield check32("alpha", raw[:, 3], ea, Bt + EPS32 * (ea.abs() + Bt))


def alpha_input_votes(W16, W32, pe, sx, raw):
    """The alpha window has to carry layer 7's accumulation bound through |w_alpha|, which is wider than the effect of
    evaluating the head on the fp16-ROUNDED layer-7 output instead of the fp32 accumulators (DESIGN.md §3).  This tells
    the two apart row by row: the fraction of rows (among those where the two models differ by more than 2^-16 of the
    head's sum of |terms|, ~30x its typical fp32 rounding) whose raw alpha lies closer to the rounded-input model.  A
    correct kernel gives ~0, the defect ~1.  Not a proof like the windows: a vote.  -> (fraction, rows counted)"""
    e7, _ = mma_ref(hidden_blocks(W16, 7, pe, sx))
    wa, ba = W32['alpha_linear.weight'][0], W32['alpha_linear.bias']
    good = e7.clamp_min(0.0) @ wa + ba
    rounded = sx[7].double() @ wa + ba
    a = raw[:, 3].double()
    sep = (good - rounded).abs() > 2.0 ** -16 * (e7.clamp_min(0.0) @ wa.abs() + ba.abs())
    closer = (a - rounded).abs() < (a - good).abs()
    return float((closer & sep).sum()) / max(1, int(sep.sum())), int(sep.sum())


def sign_words(x):
    """The ReLU sign words of a [n, C] activation plane (C = 256 or 128) as int64 [n, C/32]: word c/32, bit
    16*((c>>4)&1) + 8*(c&1) + ((c&15)>>1) is [x_c > 0] (include/neuman_b200.h, mlp_tc.cu fwd_epi)."""
    n, C = x.shape
    pos = (x.double() > 0).to(torch.int64).reshape(n, C // 32, 2, 8, 2)        # [n, word, half, pair j, even/odd]
    h = torch.arange(2, device=x.device).reshape(1, 1, 2, 1, 1)
    j = torch.arange(8, device=x.device).reshape(1, 1, 1, 8, 1)
    e = torch.arange(2, device=x.device).reshape(1, 1, 1, 1, 2)
    return (pos << (16 * h + 8 * e + j)).sum((2, 3, 4))


# ---------------------------------------------------------------------------------------------
# Layer-local references of the backward chain (csrc/mlp_tc_bwd.cu header; S = the power-of-two loss scale)
# ---------------------------------------------------------------------------------------------
def backward_checks(W16, W32, scale, d_raw, sx, sv, g_pre, g_f, g_v):
    """Yields a Check for g_v, g_f and g_pre[7..0] of nm_mlp_backward on its own inputs: the masks are (stash > 0),
    each layer's input is the kernel's own gradient plane of the layer above."""
    gs = float(scale) * d_raw.double()
    npe = n_pos(W16)
    # g_v = r16(mask_v (S g_rgb @ W_rgb)): three fp32 FMAs with fp32 weights, any order
    e, S = affine(gs[:, :3], W32['rgb_linear.weight'].T)
    yield check16("g_v", g_v, e, 3 * EPS32 * S, mask=sv > 0)
    # g_f = r16(g_v @ W16_v[:, :256]), K = 128
    e, B = mma_ref([(g_v, W16['views_linears.0.weight'][:, :256].T)])
    yield check16("g_f", g_f, e, B)
    # g_pre[7] = r16(mask_7 (g_f @ W16_f + S g_alpha w_alpha)): K = 256, then one fp32 FMA
    e, B = mma_ref([(g_f, W16['feature_linear.weight'].T)])
    e = e + gs[:, 3:4] * W32['alpha_linear.weight']
    yield check16("g_pre7", g_pre[7], e, B + EPS32 * (e.abs() + B), mask=sx[7] > 0)
    for l in range(7, 0, -1):
        w = W16[f'pts_linears.{l}.weight']
        if l == 5:
            w = w[:, npe:]
        e, B = mma_ref([(g_pre[l], w.T)])
        yield check16(f"g_pre{l - 1}", g_pre[l - 1], e, B, mask=sx[l - 1] > 0)


# ---------------------------------------------------------------------------------------------
# Encodings (Embedder.forward in float64) and the windows of the tensor-core encoder (mlp_tc.cu encode_f16)
# ---------------------------------------------------------------------------------------------
MUFU_ABS = 4e-7             # __sinf / __cosf on [-pi, pi]: 2^-21.41 absolute (CUDA programming guide)


def encoder_table(emb):
    """The fp32 frequency table the library builds (api.cu pe_table): posenc [N] frequencies, rotate [3N, 3] bvals."""
    if emb.mapping == 'rotate':
        return emb.rotate_bvals().double()
    e = torch.linspace(float(emb.min_freq), float(emb.max_freq), int(emb.N_freqs), dtype=torch.float64)
    return (2.0 ** e).float().double()


def embed64(x, emb):
    """Embedder.forward (models/vanilla.py:82-92) in float64 on fp32 inputs with the fp32 table: [n, out_dim]."""
    x = x.double()
    tab = encoder_table(emb).to(x.device)
    if emb.mapping == 'rotate':
        proj = x @ tab.T
        return torch.cat([x, torch.sin(proj), torch.cos(proj)], -1)
    out = [x]
    for f in tab:
        out += [torch.sin(x * f), torch.cos(x * f)]
    return torch.cat(out, -1)


def encoder_delta(emb):
    """Absolute error bound of one sin/cos channel of encode_f16 before its fp16 rounding: MUFU on [-pi, pi], plus the
    reduction in cycles -- posenc: one fp32 add of the residual (2^-25 cycles); rotate: two fp32 adds of three
    fractions in [-1/2, 1/2] and the residual add (4.5 * 2^-24 cycles) -- plus 2*pi's fp32 constant on |f| <= 1/2
    (8.7e-8) and the fp32 product f * 2pi (2^-24 pi)."""
    cyc = 4.5 * 2.0 ** -24 if emb.mapping == 'rotate' else 2.0 ** -25
    return MUFU_ABS + 2 * math.pi * cyc + 8.7e-8 + 2.0 ** -24 * math.pi


def encoding_check(name, v, x, emb, width):
    """nm_encode_f16's [n, width] output against r16(float64 Embedder +- delta) on the sin/cos channels, exactly r16(x) on
    the raw input channels, exactly 1 on the constant channel (= out_dim) and exactly 0 on the padding."""
    ref = embed64(x, emb)
    d = ref.shape[1]
    delta = torch.full_like(ref, encoder_delta(emb))
    delta[:, :3] = 0.0
    lo, hi = r16(ref - delta), r16(ref + delta)
    one = torch.ones(ref.shape[0], 1, dtype=torch.float64, device=ref.device)
    pad = torch.zeros(ref.shape[0], width - d - 1, dtype=torch.float64, device=ref.device)
    lo, hi = torch.cat([lo, one, pad], 1), torch.cat([hi, one, pad], 1)
    e = torch.cat([ref, one, pad], 1)
    return Check(name, v.double(), lo, hi, e, torch.cat([delta, 0 * one, pad], 1))


def pe_backward_ref(x, emb, d_enc, inv_scale=1.0):
    """The float64 Jacobian of Embedder.forward applied to d_enc [n, >= out_dim] -> (dx [n,3], B [n,3]): the bound of an
    fp32 evaluation with an accurate sincosf (2 ulp) on the fp32 argument -- exact for posenc's power-of-two frequencies,
    three fp32 FMA roundings for rotate's projection -- and nq + 1 fp32 FMAs per component, then the fp32 scale."""
    x, g = x.double(), d_enc.double()
    tab = encoder_table(emb).to(x.device)
    nf = int(emb.N_freqs)
    if emb.mapping == 'rotate':
        Bv = tab                                                   # [3N, 3]
        arg = x @ Bv.T
        arg_err = 3 * 2.0 ** -24 * (x.abs() @ Bv.abs().T)
        gs, gc = g[:, 3:3 + 3 * nf], g[:, 3 + 3 * nf:3 + 6 * nf]
    else:
        Bv = torch.zeros(3 * nf, 3, dtype=torch.float64, device=x.device)
        for k in range(nf):
            for dd in range(3):
                Bv[3 * k + dd, dd] = tab[k]
        arg = x.repeat(1, nf) * Bv.sum(1)                         # channel q = 3k + d: x_d f_k (exact in fp32)
        arg_err = torch.zeros_like(arg)
        q = torch.arange(3 * nf, device=x.device)
        k, dd = q // 3, q % 3
        gs, gc = g[:, 3 + 6 * k + dd], g[:, 6 + 6 * k + dd]
    sn, cs = torch.sin(arg), torch.cos(arg)
    w = cs * gs - sn * gc                                          # [n, 3N]
    dx = (g[:, :3] + w @ Bv) * inv_scale
    T = g[:, :3].abs() + ((cs * gs).abs() + (sn * gc).abs()) @ Bv.abs()
    arg_term = ((gs.abs() + gc.abs()) * (arg_err + 2.0 ** -23)) @ Bv.abs()
    B = abs(inv_scale) * ((3 * nf + 4) * EPS32 * T + arg_term) + EPS32 * dx.abs()
    return dx, B
