"""float64 references for the elementwise, upsample and squeeze-excite kernels of csrc/elementwise.cu (plain torch, no product
imports).

Sums are done in fp64. Where a kernel rounds a value that the result depends on before any sum, the reference restates that
rounding in fp32 and says so:
- the bilinear source coordinate and its weights (lerp_coord): computed in fp32, as PyTorch's area_pixel_compute_source_index
  does. An fp64 coordinate disagrees with a correct kernel by ~ulp(coordinate) x the neighbour difference, which at 64 -> 160 is
  far above an fp32 rounding of the result. Without align_corners the coordinate scale * (dst + 0.5) - 0.5 may be evaluated with
  one rounding (a contracting compiler's fma) or two; both restatements are formed and the allowance admits either;
- the 1 / HW scale of the pooled mean and of its gradient, and the 1 / (wh * ww) of the token-build gradient: fp32 reciprocals;
- everything that goes through expf (sigmoid, softmax) is compared at the accuracy of expf (2 ulp) on top of the fp32 roundings.
The allowance of every element is tc_ref.check's K * 2^-23 * sum|terms| (+ slack), K the longest chain of fp32 roundings in the
kernel's own summation tree (the chains are counted next to each reference).
"""
import math

import torch

from tc_ref import EPS32

GATHER_W = 24                                   # the register window of the float4 upsample gather (elementwise.cu)


def f32(v):
    return torch.tensor(v, dtype=torch.float32)


def lerp(out, inp, ac, fma=False):
    """lerp_coord for dst = 0 .. out - 1, in fp32: (i0, i1) int64 and (l0, l1) fp32. fma: the align_corners=0 coordinate with one
    rounding instead of two."""
    d = torch.arange(out, dtype=torch.float32)
    if ac:
        scale = f32(inp - 1) / f32(out - 1) if out > 1 else f32(0.0)
        src = scale * d
    else:
        scale = f32(inp) / f32(out)
        t = d + 0.5                                        # exact
        src = (scale.double() * t.double() - 0.5).float() if fma else scale * t - 0.5    # the fp64 form is exact before its rounding
        src = src.clamp_min(0.0)
    i0 = src.long().clamp_max(inp - 1)
    i1 = i0 + (i0 < inp - 1).long()
    l1 = src - i0.float()
    l0 = 1.0 - l1
    return i0, i1, l0, l1


def weights(out, inp, ac, fma=False):
    """[out, inp] fp64 matrix of the kernel's fp32 interpolation weights (the two weights of a clamped edge pixel both land on it)."""
    i0, i1, l0, l1 = lerp(out, inp, ac, fma)
    w = torch.zeros(out, inp, dtype=torch.float64)
    r = torch.arange(out)
    w.index_put_((r, i0), l0.double(), accumulate=True)
    w.index_put_((r, i1), l1.double(), accumulate=True)
    return w


def window(g, inp, out, ac):
    """lerp_window in fp32: the range [lo, hi] of destination pixels the gather visits for source cell g (int64 tensors)."""
    g = g.float()
    if ac:
        scale = f32(inp - 1) / f32(out - 1) if out > 1 else f32(0.0)
        if float(scale) <= 0.0:
            return torch.zeros_like(g, dtype=torch.long), torch.full_like(g, out - 1, dtype=torch.long)
        a, b = (g - 1.0) / scale, (g + 1.0) / scale
    else:
        inv = f32(out) / f32(inp)
        a, b = (g - 0.5) * inv - 0.5, (g + 1.5) * inv - 0.5
    lo = (torch.floor(a).long() - 1).clamp_min(0)
    hi = (torch.ceil(b).long() + 1).clamp_max(out - 1)
    return lo, hi


def max_window(inp, out, ac):
    lo, hi = window(torch.arange(inp), inp, out, ac)
    return int((hi - lo + 1).max())


def _sep(wy, wx, x, dev):
    """sum_ij wy[a, i] wx[b, j] x[n, i, j, c] in fp64 (x NHWC)."""
    wy, wx = wy.to(dev), wx.to(dev)
    t = torch.einsum('ai,nijc->najc', wy, x.double())
    return torch.einsum('bj,najc->nabc', wx, t)


def upsample_fwd_ref(x, Ho, Wo, ac):
    """(ref, mag, slack, K) of y = up(x), x [N, Hi, Wi, C]. The kernel: ly.l0 * (lx.l0 * a + lx.l1 * b) + ly.l1 * (...) (or the
    four-product form of the GPT upsample): at most 4 roundings behind each term. slack: the spread between the two
    coordinate restatements."""
    _, Hi, Wi, _ = x.shape
    refs = [_sep(weights(Ho, Hi, ac, f), weights(Wo, Wi, ac, f), x, x.device) for f in ((False, True) if not ac else (False,))]
    mag = _sep(weights(Ho, Hi, ac).abs(), weights(Wo, Wi, ac).abs(), x.abs(), x.device)
    slack = (refs[-1] - refs[0]).abs()
    return refs[0], mag, slack, 4


def upsample_bwd_ref(dy, Hi, Wi, ac):
    """(ref, mag, slack, K) of dx = up^T(dy), dy [N, Ho, Wo, C]. The gather sums, per source cell, each destination row over the
    non-zero x weights (an fma chain), then the rows (an fma chain): K = most x terms + most rows + 2 (the weight of a clamped edge
    pixel is an fp32 sum of two)."""
    _, Ho, Wo, _ = dy.shape
    out = []
    for f in ((False, True) if not ac else (False,)):
        wy, wx = weights(Ho, Hi, ac, f), weights(Wo, Wi, ac, f)
        out.append(_sep(wy.t(), wx.t(), dy, dy.device))
    wy, wx = weights(Ho, Hi, ac), weights(Wo, Wi, ac)
    mag = _sep(wy.t().abs(), wx.t().abs(), dy.abs(), dy.device)
    K = int((wx != 0).sum(0).max()) + int((wy != 0).sum(0).max()) + 2
    return out[0], mag, (out[-1] - out[0]).abs(), K


def slab_view(tok, t_off, gh, gw):
    """The token slab [N, G, C] of rows t_off .. t_off + G, *viewed* as [N, C, gh, gw] (transfuser.py:363-364), returned NHWC
    [N, gh, gw, C]."""
    N, _, C = tok.shape
    G = gh * gw
    return tok[:, t_off:t_off + G].reshape(N, C, gh, gw).permute(0, 2, 3, 1)


def fp32_recip(n):
    """1.f / (float)n, the kernels' fp32 scale (exact restatement)."""
    return float(f32(1.0) / f32(float(n)))


def pool_splits(HW):
    """Splits of pool_hw_kernel (tfb_pool_hw_fwd, and tfb_se_bwd_reduce's grid form)."""
    return min(32, (HW + 255) // 256)


def pool_terms(HW):
    """pool_hw_kernel: each thread sums its pixels p = split * 8 + row phase (step splits * 8), the 8 row phases are added, the
    splits are added in order, the scale: the longest fp32 chain."""
    s = pool_splits(HW)
    return math.ceil(HW / (s * 8)) + 8 + s + 1


def se_reduce_flat(HW, C):
    return C // 4 <= 128 and HW >= 1024


def se_reduce_terms(N, HW, C, sms):
    """tfb_se_bwd_reduce: the flat kernel (C / 4 <= 128, HW >= 1024) with the split count of the host (>= 16 rows per thread,
    capped at 4 * SMs / N): rows per thread, the RPB row phases, the splits; else pool_hw_kernel."""
    if not se_reduce_flat(HW, C):
        return pool_terms(HW)
    rpb = 256 // (C // 4)
    sp = (HW + rpb * 16 - 1) // (rpb * 16)
    sp = max(1, min(sp, (4 * sms + N - 1) // N))
    return math.ceil(HW / (sp * rpb)) + rpb + sp + 1


def sigmoid_ref(x):
    """(ref, mag, K): expf (2 ulp), the add and the division, each relative to y."""
    y = torch.sigmoid(x.double())
    return y, y, 4


def softmax_ref(S, scale):
    """Row softmax of fl32(S * scale) (the product the kernel rounds before its max): (P, mag, slack, K). The argument x - m of expf
    is rounded once more (or the product is contracted into it), expf is within 2 ulp, each lane sums ceil(L / 32) values and the
    warp adds 5 levels, then 1 / sum and the product: K = ceil(L / 32) + 5 + 4 relative to P, and slack = P * EPS32 * (|x - m| + |x|)
    for the rounding of the argument, and the same of the row's worst element for the sum."""
    L = S.shape[-1]
    x = (S.float() * f32(scale).to(S.device)).double()
    m = x.max(-1, keepdim=True).values
    P = torch.softmax(x, -1)
    argerr = EPS32 * ((x - m).abs() + x.abs())
    slack = P * (argerr + argerr.max(-1, keepdim=True).values)
    return P, P, slack, math.ceil(L / 32) + 5 + 4


def softmax_bwd_ref(P, dPd, scale):
    """dS = scale * P * (g - sum_j g_j P_j) in fp64 from the kernel's inputs: (ref, mag, K). The dot is a ceil(L / 32) fma chain per
    lane and a 5-level warp sum; then the difference and two products."""
    L = P.shape[-1]
    p, g = P.double(), dPd.double()
    dot = (g * p).sum(-1, keepdim=True)
    ref = scale * p * (g - dot)
    mag = (scale * p).abs() * (g.abs() + (g * p).abs().sum(-1, keepdim=True))
    return ref, mag, math.ceil(L / 32) + 5 + 4


def se_mlp_bwd_ref(dgate, gate, h, pooled, w1, w2):
    """The squeeze-excite MLP backward in fp64: dict of (ref, mag, K) per output. Chains (tfb_se_mlp_bwd): ds = dgate * g * (1 - g)
    (3 roundings); db2 and dw2 are N-term chains on ds; dh = (h > 0) * sum over the chunks (16-channel fma chains, then the chunks in
    order) of ds w2; db1 and dw1 are N-term chains on dh; dpool sums each of the 16 slices of Cr (ceil(Cr / 16) fmas) and the
    slices in order."""
    N, C = dgate.shape
    Cr = h.shape[1]
    g = gate.double()
    ds = dgate.double() * g * (1 - g)
    dsm = ds.abs()
    keep = (h > 0).double()
    w1d, w2d, hd, pd = w1.double(), w2.double(), h.double(), pooled.double()
    dh = keep * (ds @ w2d)
    dhm = keep * (dsm @ w2d.abs())
    k_dh = 3 + 16 + math.ceil(C / 16)
    return dict(
        db2=(ds.sum(0), dsm.sum(0), 3 + N),
        dw2=(ds.t() @ hd, dsm.t() @ hd.abs(), 3 + N + 1),
        db1=(dh.sum(0), dhm.sum(0), k_dh + N),
        dw1=(dh.t() @ pd, dhm.t() @ pd.abs(), k_dh + N + 1),
        dpool=(dh @ w1d, dhm @ w1d.abs(), k_dh + math.ceil(Cr / 16) + 16 + 1))
