"""Exact-operand references for the bf16 tensor-core kernels (plain torch, no product imports).

The kernels round their operands to bf16 and accumulate in fp32. A reference that rounds the SAME operands the same way and
contracts in fp64 differs from the kernel only by the fp32 accumulation order, so it can be compared element by element:
|out - ref| <= K * 2^-23 * (|A| |B|) is the worst-case fp32 bound of a K-term sum (2u per add, valid even for truncating adders).
A wrong row, a missing k-block, a mis-staged chunk or a skipped store is orders of magnitude above that bound.

The attention reference restates the rounding points of csrc/attn_tc.cu. Where the kernel rounds an intermediate it computed
itself (the probabilities / score gradients, the bf16 A operand of its second product), fp32 exp2f against fp64 exp can land on
the other side of a bf16 rounding midpoint. Those roundings are tracked: an element whose exact value lies within its own error
bound of a midpoint may round to either neighbour, and one bf16 ulp of it times |B| is added to the element-wise allowance.
"""
import math

import torch

U32 = 0xFFFFFFFF
EPS32 = 2.0 ** -23          # 2u of fp32 (u = 2^-24): the per-add bound used throughout
TINY = 1e-30
SENT = -1024.0              # sentinel behind every Guarded output (exactly representable in bf16 and fp32)


def bf(x):
    """x rounded to bf16 (round-to-nearest-even, as __floats2bfloat162_rn and torch's cast) and widened to fp64."""
    return x.bfloat16().double()


def bf16_ulp(x):
    """Spacing of bf16 values at |x| (fp64): 2^(floor(log2|x|) - 7); the subnormal spacing below 2^-126."""
    a = x.abs().double().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def bf_flip(x, err):
    """(bf16(x), flip) where flip is one bf16 ulp wherever x lies within err of a rounding midpoint (a value computed to within err
    may round to the other neighbour there) and 0 elsewhere."""
    r = bf(x)
    ulp = bf16_ulp(x)
    lo = torch.where(r > x, r - ulp, r)            # the bf16 neighbours bracketing x (r is one of them)
    dist = ((x - (lo + ulp / 2)).abs())
    return r, torch.where(dist <= err, bf16_ulp(torch.maximum(x.abs(), r.abs())), torch.zeros_like(x))


def contract(a, b, rounding=True):
    """a [..., M, K] @ b [..., K, N] with both operands rounded to bf16 (rounding=False: as given), in fp64.
    Returns (result, |a| @ |b|)."""
    a = bf(a) if rounding else a.double()
    b = bf(b) if rounding else b.double()
    return a @ b, a.abs() @ b.abs()


def check(out, ref, mag, K, tol, slack=None, what='', floor=0.0):
    """out (kernel) against ref (fp64): every element finite; relative L2 <= tol (the norm of ref floored at `floor`, for outputs
    that are zero up to rounding); |out - ref| <= K * 2^-23 * mag (+ slack) + tiny.
    Returns (relative L2, worst element-wise ratio |out - ref| / allowance)."""
    o = out.double()
    ref = ref.double()
    assert o.shape == ref.shape, (what, o.shape, ref.shape)
    assert torch.isfinite(o).all(), '%s: %d non-finite elements' % (what, int((~torch.isfinite(o)).sum()))
    err = (o - ref).abs()
    allow = K * EPS32 * mag.double() + TINY
    if slack is not None:
        allow = allow + slack.double()
    ratio = (err / allow).max().item() if err.numel() else 0.0
    rel = (err.norm() / ref.norm().clamp_min(max(floor, TINY))).item()
    if ratio > 1.0:
        i = int((err / allow).flatten().argmax())
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), err.shape))
        raise AssertionError('%s: element %s = %.9g, reference %.9g, |diff| %.3g > allowance %.3g (%d elements over; rel L2 %.3g)'
                             % (what, idx, o[idx].item(), ref[idx].item(), err[idx].item(), allow[idx].item(),
                                int((err > allow).sum()), rel))
    assert rel <= tol, '%s: relative L2 %.3g > %.3g' % (what, rel, tol)
    return rel, ratio


class Guarded:
    """A NaN-filled output tensor followed by sentinel elements that must stay bit-unchanged."""

    def __init__(self, shape, dtype, device='cuda'):
        n = math.prod(shape)
        self.buf = torch.empty(n + 64, dtype=dtype, device=device)
        self.t = self.buf[:n].view(shape)
        self.n = n

    def reset(self):
        self.buf[self.n:].fill_(SENT)
        self.t.fill_(float('nan'))
        return self.t

    def tail_ok(self):
        return bool((self.buf[self.n:] == SENT).all())

    def bits(self):
        return self.buf.clone().view(torch.int16 if self.buf.dtype == torch.bfloat16 else torch.int32)


# ------------------------------------------------------------------ attention dropout mask (csrc/attn_tc.cu drop_scale)
def _mul32(x, c):
    """(x * c) mod 2^32 for int64 tensors x < 2^32 and a constant c < 2^32, without int64 overflow."""
    return (x * (c & 0xFFFF) + (((x * (c >> 16)) & 0xFFFF) << 16)) & U32


def keep_mask(seed, idx, p):
    """The kernel's keep decision for counter idx (int64 tensor, taken mod 2^32) under the 64-bit seed (*seed_dev + seed_off):
    a 32-bit hash, its top 24 bits as u in [0, 1), keep when NOT (u < p) in float32."""
    seed &= (1 << 64) - 1
    lo, hi = seed & U32, seed >> 32
    x = (_mul32(idx & U32, 0x9E3779B1) + lo) & U32
    x = x ^ (x >> 16)
    x = _mul32(x, 0x85EBCA6B)
    x = x ^ hi
    x = x ^ (x >> 13)
    x = _mul32(x, 0xC2B2AE35)
    x = x ^ (x >> 16)
    u = (x >> 8).to(torch.float32) * (1.0 / 16777216.0)
    return ~(u < torch.tensor(p, dtype=torch.float32))


def keep_scale(p):
    """1 / (1 - p) in float32 (the kernel's keep scale), 1 when p == 0."""
    if p <= 0:
        return 1.0
    one = torch.tensor(1.0, dtype=torch.float32)
    return float(one / (one - torch.tensor(p, dtype=torch.float32)))


def drop_factor(seed, B, nh, T, p, device='cpu'):
    """[B, nh, T(query i), T(key j)] fp64 dropout factor (0 or keep_scale(p)) at counter ((b*nh + h)*T + i)*T + j."""
    if p <= 0:
        return torch.ones((B, nh, T, T), dtype=torch.float64, device=device)
    idx = torch.arange(B * nh * T * T, dtype=torch.int64, device=device).view(B, nh, T, T)
    return keep_mask(seed, idx, p).double() * keep_scale(p)


# ------------------------------------------------------------------ attention
def split_heads(qkv, B, T, nh, hs):
    """[B*T, 3C] packed q | k | v -> three [B, nh, T, hs] fp64 tensors."""
    C = nh * hs
    x = qkv.double().view(B, T, 3, nh, hs)
    return [x[:, :, i].permute(0, 2, 1, 3) for i in range(3)]


def merge_heads(x):
    """[B, nh, T, hs] -> [B*T, nh*hs]."""
    B, nh, T, hs = x.shape
    return x.permute(0, 2, 1, 3).reshape(B * T, nh * hs)


def attn_fwd_ref(qkv, B, T, nh, hs, scale, drop, rounding=True):
    """Forward at the kernel's rounding points. drop: [B, nh, T, T] factor (drop_factor). Returns a dict with
    y [B*T, C], lse [B, nh, T] and the allowances (y_mag, y_slack, y_K, lse_slack) for check()."""
    q, k, v = split_heads(qkv, B, T, nh, hs)
    rnd = bf if rounding else (lambda t: t)
    q, k, v = rnd(q), rnd(k), rnd(v)
    S = q @ k.transpose(-1, -2)
    Smag = q.abs() @ k.abs().transpose(-1, -2)
    mx = S.max(-1, keepdim=True).values
    e = torch.exp(scale * (S - mx))
    ssum = e.sum(-1, keepdim=True)                                   # before dropout
    x = e * drop
    # error of the kernel's fp32 e: the scores (hs-term fp32 sums, also in the row max), exp2f of an fp32 argument, the keep scale
    errS = hs * EPS32 * Smag
    errS_row = errS.max(-1, keepdim=True).values
    arg = (scale * (S - mx)).abs()
    err_x = x * (scale * (errS + errS_row) * 1.01 + (arg + 4.0) * 4 * EPS32)
    if rounding:
        A, flip = bf_flip(x, err_x)
    else:
        A, flip = x, torch.zeros_like(x)
    num = A @ v
    num_mag = A.abs() @ v.abs()
    y = num / ssum
    # 1 / sum: a T-term fp32 sum of values each within err_e of the exact e; the product with 1/sum is two more roundings
    err_sum = (T * EPS32 * ssum + (err_x / drop.clamp_min(1.0)).sum(-1, keepdim=True))
    rel_sum = err_sum / ssum
    y_slack = (flip @ v.abs()) / ssum + num_mag / ssum * (rel_sum * 1.01 + 4 * EPS32)
    lse = scale * mx.squeeze(-1) + torch.log(ssum.squeeze(-1))
    lse_slack = scale * errS_row.squeeze(-1) + rel_sum.squeeze(-1) + 8 * EPS32 * lse.abs() + 1e-7
    return dict(y=merge_heads(y), y_mag=merge_heads(num_mag / ssum), y_slack=merge_heads(y_slack), y_K=T,
                lse=lse, lse_slack=lse_slack)


def attn_bwd_ref(qkv, dy, y, lse, B, T, nh, hs, scale, drop, rounding=True):
    """Backward at the kernel's rounding points, from the forward's y (fp32 or its bf16 copy, as the kernel was given it) and
    lse. Returns dict with dqkv [B*T, 3C] and its allowances (mag, slack, K) for check()."""
    q, k, v = split_heads(qkv, B, T, nh, hs)
    rnd = bf if rounding else (lambda t: t)
    q, k, v = rnd(q), rnd(k), rnd(v)
    C = nh * hs
    dy4 = dy.double().view(B, T, nh, hs).permute(0, 2, 1, 3)
    y4 = y.double().view(B, T, nh, hs).permute(0, 2, 1, 3)
    D = (dy4 * y4).sum(-1, keepdim=True)
    errD = hs * EPS32 * (dy4 * y4).abs().sum(-1, keepdim=True)
    dO = rnd(dy4)
    lse = lse.double().unsqueeze(-1)
    S = q @ k.transpose(-1, -2)
    errS = hs * EPS32 * (q.abs() @ k.abs().transpose(-1, -2))
    P = torch.exp(scale * S - lse)
    errP = P * (scale * errS * 1.01 + ((scale * S).abs() + lse.abs() + 4.0) * 4 * EPS32)
    dPd = dO @ v.transpose(-1, -2)
    errdP = hs * EPS32 * (dO.abs() @ v.abs().transpose(-1, -2))
    Pd = P * drop
    g = dPd * drop - D
    dS = scale * P * g
    err_Pd = errP * drop
    err_dS = scale * (errP * g.abs() + P * (errdP * drop + errD) * 1.01) + dS.abs() * 4 * EPS32
    if rounding:
        Pd_b, fPd = bf_flip(Pd, err_Pd)
        dS_b, fdS = bf_flip(dS, err_dS)
    else:
        Pd_b, fPd, dS_b, fdS = Pd, torch.zeros_like(Pd), dS, torch.zeros_like(dS)
    dQ = dS_b @ k
    dK = dS_b.transpose(-1, -2) @ q
    dV = Pd_b.transpose(-1, -2) @ dO
    mags = [dS_b.abs() @ k.abs(), dS_b.abs().transpose(-1, -2) @ q.abs(), Pd_b.abs().transpose(-1, -2) @ dO.abs()]
    slacks = [fdS @ k.abs(), fdS.transpose(-1, -2) @ q.abs(), fPd.transpose(-1, -2) @ dO.abs()]
    cat = lambda ts: torch.cat([merge_heads(t) for t in ts], dim=1)
    return dict(dqkv=cat([dQ, dK, dV]), mag=cat(mags), slack=cat(slacks), K=T, D=D.squeeze(-1))


def attn_plain(qkv, B, T, nh, hs, scale, drop):
    """Plain fp64 attention on the inputs as given (no rounding): y = (softmax(scale q k^T) * drop) v, with autograd."""
    q, k, v = split_heads(qkv, B, T, nh, hs)
    q, k, v = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    y = (torch.softmax(scale * q @ k.transpose(-1, -2), dim=-1) * drop) @ v
    return merge_heads(y), (q, k, v), y


def attn_plain_grads(qkv, dy, B, T, nh, hs, scale, drop):
    """fp64 autograd dq | dk | dv of attn_plain for output gradient dy [B*T, C], packed as [B*T, 3C]."""
    _, (q, k, v), y = attn_plain(qkv, B, T, nh, hs, scale, drop)
    dy4 = dy.double().view(B, T, nh, hs).permute(0, 2, 1, 3)
    gq, gk, gv = torch.autograd.grad(y, (q, k, v), dy4)
    return torch.cat([merge_heads(t) for t in (gq, gk, gv)], dim=1)


# ------------------------------------------------------------------ convolution
def conv3x3_ref(x, w, bias, stride, groups, dy=None):
    """fp64 3x3 conv (pad 1) of bf16-rounded NHWC x [N,H,W,Cin] and w [Cout, Cin/groups, 3, 3]; with dy (NHWC) also its input and
    weight gradients on bf16-rounded dy. Returns NHWC y (+ bias), |x| * |w|, and (dx, |dy| * |w|, dw, |x| * |dy|) when dy is given."""
    import torch.nn.functional as F
    xn, wr = bf(x).permute(0, 3, 1, 2), bf(w)
    y = F.conv2d(xn, wr, None, stride=stride, padding=1, groups=groups)
    mag = F.conv2d(xn.abs(), wr.abs(), None, stride=stride, padding=1, groups=groups)
    if bias is not None:
        y = y + bias.double().view(1, -1, 1, 1)
        mag = mag + bias.double().abs().view(1, -1, 1, 1)
    nhwc = lambda t: t.permute(0, 2, 3, 1)
    if dy is None:
        return nhwc(y), nhwc(mag)
    gn = bf(dy).permute(0, 3, 1, 2)
    dx = torch.nn.grad.conv2d_input(xn.shape, wr, gn, stride=stride, padding=1, groups=groups)
    dx_mag = torch.nn.grad.conv2d_input(xn.shape, wr.abs(), gn.abs(), stride=stride, padding=1, groups=groups)
    dw = torch.nn.grad.conv2d_weight(xn, wr.shape, gn, stride=stride, padding=1, groups=groups)
    dw_mag = torch.nn.grad.conv2d_weight(xn.abs(), wr.shape, gn.abs(), stride=stride, padding=1, groups=groups)
    return nhwc(y), nhwc(mag), nhwc(dx), nhwc(dx_mag), dw, dw_mag


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(TINY)).item()


def scale_for(hs):
    return 1.0 / math.sqrt(hs)
