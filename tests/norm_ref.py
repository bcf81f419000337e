"""float64 references for the normalisation kernels of csrc/norm.cu (plain torch, no product imports).

Statistics are compared with a two-pass fp64 mean and biased variance. Every column reduction of norm.cu sums at most 64 terms per
thread in fp32 before the sum moves to fp64, so
    |mean - ref| <= 64 * 2^-23 * mean|x| + 1/2 ulp
    |invstd / ref - 1| <= 32 * 2^-23 * E[x^2] / (var + eps) + 2^-24.
E[x^2] / var = 1 + (mean / std)^2: the error of E[x^2] - E[x]^2 grows with the square of the offset, and the bound says so.

Outputs (y, dx, the pooled means, LayerNorm's y / dx) are compared element by element with an fp64 evaluation that takes the
statistics the kernel published itself (save_mean / save_invstd, dgamma / dbeta, save_mean / save_rstd), at an allowance of a few
fp32 roundings of the magnitudes of the terms (tc_ref.check). A wrong channel, row, slab or split is then orders of magnitude over
the allowance, and an error of the statistics shows only in the statistics check. ReLU masks are evaluated exactly and must agree
bit for bit.
"""
import math

import torch

from tc_ref import EPS32, check

U24 = 2.0 ** -24
STAT_TERMS = 64             # fp32 partial length of every colreduce* kernel


def ulp32(x):
    """Spacing of fp32 values at |x| (fp64)."""
    a = x.abs().double().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 23)


def moments(x):
    """Two-pass fp64 mean, biased variance, E[x^2] and mean|x| over the rows of x [M, C]."""
    xd = x.double()
    mean = xd.mean(0)
    var = ((xd - mean) ** 2).mean(0)
    return mean, var, (xd * xd).mean(0), xd.abs().mean(0)


def check_stats(mean_k, invstd_k, x, eps, what=''):
    """The kernel's fp32 save_mean / save_invstd against the two-pass fp64 values at the partial-length bound (module docstring).
    Returns (worst mean ratio, worst invstd ratio, worst relative invstd error)."""
    mean, var, ex2, mabs = moments(x)
    ref_is = 1.0 / torch.sqrt(var + eps)
    allow_m = STAT_TERMS * EPS32 * mabs + 0.5 * ulp32(mean) + 1e-30
    err_m = (mean_k.double() - mean).abs()
    rm = (err_m / allow_m).max().item()
    assert rm <= 1.0, '%s: mean off by %.3g x its allowance at channel %d' % (what, rm, int((err_m / allow_m).argmax()))
    rel = (invstd_k.double() / ref_is - 1.0).abs()
    allow_i = STAT_TERMS / 2 * EPS32 * ex2 / (var + eps) + U24
    ri = (rel / allow_i).max().item()
    assert ri <= 1.0, '%s: invstd off by %.3g x its allowance at channel %d' % (what, ri, int((rel / allow_i).argmax()))
    return rm, ri, rel.max().item()


def stats_from_sums(s0, s1, N, eps):
    """save_mean / save_invstd as the kernels publish them from fp64 sums (bn_publish): fp64 arithmetic rounded to fp32 once."""
    mean = s0 / N
    var = (s1 / N - mean * mean).clamp_min(0.0)
    return mean.float(), (1.0 / torch.sqrt(var + eps)).float()


def xhat32(x, mean, invstd):
    """x-hat at the kernels' rounding points: fl32(fl32(x - mean) * invstd)."""
    return (x.float() - mean.float()) * invstd.float()


def relu_mask(x, mean, invstd, gamma, beta):
    """The kernels' ReLU mask fmaf(xhat, gamma, beta) > 0, evaluated exactly: the product of two fp32 values is exact in fp64 and
    the rounding of the sum keeps its sign."""
    return xhat32(x, mean, invstd).double() * gamma.double() + beta.double() > 0


def bn_y_direct(x, mean, invstd, gamma, beta, relu, res=None):
    """(x - mean) * invstd * gamma + beta (+ residual) (ReLU) in fp64 from the given fp32 statistics, with (mag, K) for check()."""
    d = (x.double() - mean.double()) * invstd.double()
    z = d * gamma.double() + beta.double()
    mag = (d * gamma.double()).abs() + beta.double().abs()
    if res is not None:
        z = z + res.double()
        mag = mag + res.double().abs()
    return (torch.relu(z) if relu else z), mag, 5


def bn_y_scsh(x, mean, invstd, gamma, beta, relu, res=None):
    """x * sc + sh with sc = fl32(gamma * invstd), sh = fl32(fma(-mean, sc, beta)) (the kernels that read statistics), in fp64."""
    sc = (gamma.float() * invstd.float()).double()
    sh = (-mean.double() * sc + beta.double()).float().double()
    z = x.double() * sc + sh
    mag = (x.double() * sc).abs() + sh.abs() + (mean.double() * sc).abs() + beta.double().abs()
    if res is not None:
        z = z + res.double()
        mag = mag + res.double().abs()
    return (torch.relu(z) if relu else z), mag, 4


def pool_terms(HW, C, flat):
    """Longest chain of fp32 additions behind one pooled mean (bn_apply_pool*_kernel): rows per thread, the row phases of a block,
    the splits of the ordered sum, the scaling. Independent of the SM count (splits >= 1)."""
    if flat:
        rpb = 256 // (C // 4)
        return math.ceil(HW / rpb) + rpb + math.ceil(HW / (rpb * 16)) + 2
    splits = min(32, (HW + 255) // 256)
    return math.ceil(HW / (splits * 8)) + 8 + splits + 2


def pooled_ref(y, n, HW, C):
    """Per-sample mean over the HW pixels of the kernel's own y, in fp64, and its magnitude."""
    yd = y.double().view(n, HW, C)
    return yd.mean(1), yd.abs().mean(1)


def bn_bwd_ref(x, g, mask, mean, invstd, gmag=None):
    """fp64 dbeta = sum g, dgamma = sum g * xhat over the rows (g: the gradient of the BatchNorm output, mask applied here), with
    their magnitudes; xhat from the kernel's statistics. gmag: |g| before cancellation (the squeeze-excite gradient)."""
    keep = mask.double() if mask is not None else torch.ones_like(g, dtype=torch.float64)
    g = g.double() * keep
    gmag = (gmag.double() if gmag is not None else g.abs()) * keep
    xh = (x.double() - mean.double()) * invstd.double()
    return dict(g=g, gmag=gmag, xh=xh, dbeta=g.sum(0), dgamma=(g * xh).sum(0), mb=gmag.sum(0), mg=(gmag * xh.abs()).sum(0))


def bn_dx_ref(r, gamma, invstd, dgamma_k, dbeta_k, M):
    """dx = gamma * invstd * (g - dbeta / M - xhat * dgamma / M) from the kernel's own dgamma / dbeta, with (mag, K)."""
    gi = gamma.double() * invstd.double()
    mb, mg = dbeta_k.double() / M, dgamma_k.double() / M
    dx = gi * (r['g'] - mb - r['xh'] * mg)
    mag = gi.abs() * (r['gmag'] + mb.abs() + (r['xh'] * mg).abs())
    return dx, mag, 8


def ln_fwd_ref(x, mean_k, rstd_k, gamma, beta):
    """LayerNorm y from the kernel's own per-row mean / rstd, (mag, K)."""
    d = (x.double() - mean_k.double()[:, None]) * rstd_k.double()[:, None]
    return d * gamma.double() + beta.double(), (d * gamma.double()).abs() + beta.double().abs(), 5


def ln_block_terms(C):
    """fp32 additions behind one block_sum over a row of C: C / 256 per thread, 5 warp levels, 3 levels of the 8 warps, the divide."""
    return math.ceil(C / 256) + 10


def check_ln_stats(mean_k, rstd_k, x, eps, what=''):
    """LayerNorm's fp32 row mean and rstd (two fp32 passes, rsqrtf) against fp64. Returns the worst ratios."""
    C = x.shape[1]
    xd = x.double()
    mean = xd.mean(1)
    var = ((xd - mean[:, None]) ** 2).mean(1)
    K = ln_block_terms(C)
    allow_m = K * EPS32 * xd.abs().mean(1) + 0.5 * ulp32(mean) + 1e-30
    rm = ((mean_k.double() - mean).abs() / allow_m).max().item()
    assert rm <= 1.0, '%s: row mean off by %.3g x its allowance' % (what, rm)
    # var from the fp32 mean: + (mean - mean_k)^2; fp32 differences (one rounding of |x|), squares and the K-term sum
    dm = (mean_k.double() - mean).abs()
    var_err = (K + 4) * EPS32 * var + 2 * EPS32 * (xd.abs() * (xd - mean[:, None]).abs()).mean(1) + dm * dm
    allow_r = 0.5 * var_err / (var + eps) + 4 * EPS32           # + rsqrtf (2 ulp) and the rounding of the sum with eps
    rel = (rstd_k.double() * torch.sqrt(var + eps) - 1.0).abs()
    rr = (rel / allow_r).max().item()
    assert rr <= 1.0, '%s: rstd off by %.3g x its allowance at row %d' % (what, rr, int((rel / allow_r).argmax()))
    return rm, rr


def ln_dx_ref(x, dy, gamma, mean_k, rstd_k):
    """LayerNorm dx from the kernel's own mean / rstd: rstd * (gg - mean_c(gg) - xhat * mean_c(gg * xhat)), gg = dy * gamma; (mag, K)."""
    C = x.shape[1]
    r = rstd_k.double()[:, None]
    xh = (x.double() - mean_k.double()[:, None]) * r
    gg = dy.double() * gamma.double()
    m1, m2 = gg.mean(1, keepdim=True), (gg * xh).mean(1, keepdim=True)
    dx = r * (gg - m1 - xh * m2)
    mag = r * (gg.abs() + gg.abs().mean(1, keepdim=True) + xh.abs() * (gg * xh).abs().mean(1, keepdim=True))
    return dx, mag, ln_block_terms(C) + 6


def ln_param_ref(x, dy, mean_k, rstd_k):
    """dbeta = sum_r dy, dgamma = sum_r dy * xhat (xhat from the kernel's row statistics) in fp64, with magnitudes."""
    xh = (x.double() - mean_k.double()[:, None]) * rstd_k.double()[:, None]
    g = dy.double()
    return dict(dbeta=g.sum(0), dgamma=(g * xh).sum(0), mb=g.abs().sum(0), mg=(g * xh).abs().sum(0))


def ln_param_terms(R):
    """fp32 additions behind one LayerNorm dgamma / dbeta partial: rows per thread (<= 64 splits of 8 row phases), the 8 phases, and
    the rounding points of xhat."""
    splits = max(1, min(64, math.ceil(R / 64)))
    return math.ceil(R / (splits * 8)) + 8 + 6


def colreduce_splits(M, slabs, sms, min_rows=16):
    """Row splits of the 2-D column reductions (colreduce_splits in norm.cu)."""
    want = (4 * sms + slabs - 1) // slabs
    want = min(want, math.ceil(M / (8 * min_rows)))
    return max(1, min(want, 65535))


def grad_prep_terms(M, C, sms):
    """fp32 additions behind one dbias of tfb_grad_prep: it accumulates every row of its split in fp32 (no 64-row cap), then 8 row
    phases; the split partials are added in fp64."""
    splits = colreduce_splits(M, (C + 31) // 32, sms)
    return math.ceil(M / (splits * 8)) + 8 + 2

