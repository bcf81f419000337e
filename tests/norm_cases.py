"""Cases of the normalisation kernels (csrc/norm.cu), shared by tests/test_norm_exact.py (H100, full sizes) and
tests/test_norm_emulated.py (CPU emulation, reduced sizes that still cross every dispatch boundary). Every case:
- runs twice into NaN-filled, sentinel-guarded outputs (tc_ref.Guarded), and the two runs give the same bits;
- leaves the sums_ws workspace all zero after every call;
- compares its outputs with the float64 references of tests/norm_ref.py.
A case returns {check: worst allowance ratio} for the caller to print."""
import math

import pytest
import torch

import norm_ref as N
from tc_ref import Guarded

EPS = float(torch.tensor(1e-5, dtype=torch.float32))     # the fp32 eps the kernels take, as a Python float (exact)
MOM = 0.1
TOL = 1e-3                # relative L2: a backstop only, the element-wise allowance is the check
SEED = 0x5EED0F00D


class Ctx:
    def __init__(self, call, dev, sms):
        self.call, self.dev, self.sms = call, dev, sms
        self.ws = torch.zeros(2 * 8192 + 8, dtype=torch.float64, device=dev)
        self.res = {}

    def rand(self, shape, seed, scale=1.0, shift=0.0):
        g = torch.Generator(device=self.dev).manual_seed(seed)
        return torch.randn(shape, generator=g, device=self.dev) * scale + shift

    def affine(self, C, seed):
        """gamma around 1 with some negative channels, beta around 0: ReLU masks of every kind."""
        return self.rand((C,), seed, 0.6, 0.8), self.rand((C,), seed + 1, 0.4)

    def out(self, shape, dtype=torch.float32):
        return Guarded(shape, dtype, self.dev)

    def sync(self):
        if self.dev == 'cuda' or (isinstance(self.dev, torch.device) and self.dev.type == 'cuda'):
            torch.cuda.synchronize()

    def __call__(self, name, *args):
        """One entry-point call; afterwards the workspace must be all zero again."""
        self.call(name, *args)
        self.sync()
        assert not bool(self.ws.any()), '%s left sums_ws non-zero' % name

    def twice(self, launch, outs, pre=None):
        """Runs launch() twice into reset outputs: every sentinel intact, the same bits both times."""
        runs = []
        for _ in range(2):
            for o in outs:
                o.reset()
            if pre is not None:
                pre()
            launch()
            self.sync()
            assert all(o.tail_ok() for o in outs), 'write past the end of an output'
            runs.append([o.bits() for o in outs])
        self.last = runs[0]
        for i, (a, b) in enumerate(zip(*runs)):
            assert torch.equal(a, b), 'output %d differs between two launches' % i

    def check(self, name, out, ref, mag, K, floor_frac=1e-3, slack=None):
        rel, ratio = N.check(out, ref, mag, K, TOL, slack, name, floor=floor_frac * mag.double().norm().item())
        self.res[name] = max(self.res.get(name, 0.0), ratio)
        return ratio

    def note(self, name, v):
        self.res[name] = max(self.res.get(name, 0.0), v)


def bits_equal(a, b, what):
    a, b = a.contiguous(), b.contiguous()
    view = torch.int16 if a.dtype == torch.bfloat16 else torch.int32
    ne = a.view(view) != b.view(view)
    assert not bool(ne.any()), '%s: %d elements differ, first at %s' % (what, int(ne.sum()), tuple(int(i) for i in ne.nonzero()[0]))


def mask_equal(k, ref, what):
    ne = k != ref
    assert not bool(ne.any()), '%s: ReLU mask differs at %d elements, first at %s' % (what, int(ne.sum()), tuple(int(i) for i in ne.nonzero()[0]))


def _stats_fp64(x):
    return torch.cat([x.double().sum(0), (x.double() ** 2).sum(0)])


# ------------------------------------------------------------------ tfb_bn_fwd + tfb_bn_bwd
BN_VARIANTS = ('relu', 'plain', 'residual', 'y16')


def bn_train(c, C, M, shift, variant, seed=0):
    """tfb_bn_fwd then tfb_bn_bwd. variant: relu (mask recomputed in backward), plain, residual (relu(bn(x) + res), ymask +
    gmasked backward), y16 (relu, bf16 sidecars y16 / dx16)."""
    x = c.rand((M, C), seed, 1.0, shift)
    gamma, beta = c.affine(C, seed + 1)
    dy = c.rand((M, C), seed + 3)
    res = c.rand((M, C), seed + 4) if variant == 'residual' else None
    relu = variant != 'plain'
    side = variant == 'y16'
    y, mean, invstd = c.out((M, C)), c.out((C,)), c.out((C,))
    y16, dx16 = (c.out((M, C), torch.bfloat16), c.out((M, C), torch.bfloat16)) if side else (None, None)
    dx, dg, db = c.out((M, C)), c.out((C,)), c.out((C,))
    gm = c.out((M, C)) if res is not None else None
    rm, rv = torch.zeros(C, device=c.dev), torch.ones(C, device=c.dev)

    def pre():
        rm.zero_()
        rv.fill_(1.0)

    def launch():
        c('tfb_bn_fwd', x, y.t, M, C, gamma, beta, EPS, MOM, int(relu), rm, rv, mean.t, invstd.t, c.ws, y16 and y16.t, res, None, 0)
        c('tfb_bn_bwd', x, dy, dx.t, M, C, gamma, beta, mean.t, invstd.t, int(relu and res is None), dg.t, db.t, c.ws, dx16 and dx16.t,
          y.t if res is not None else None, gm and gm.t)
    outs = [o for o in (y, mean, invstd, y16, dx, dg, db, dx16, gm) if o is not None]
    c.twice(launch, outs, pre)

    _, ri, rel = N.check_stats(mean.t, invstd.t, x, EPS, 'stats C %d M %d shift %g' % (C, M, shift))
    c.note('invstd', ri)
    c.note('invstd rel err, mean/std %g' % shift, rel)
    # running statistics: rm from the published mean (same fp32 operations), rv against the fp64 unbiased variance
    bits_equal(rm, torch.tensor(MOM, dtype=torch.float32) * mean.t, 'running_mean')
    _, var, ex2, _ = N.moments(x)
    unb = var * M / (M - 1) if M > 1 else var
    rv_ref = (1 - MOM) + MOM * unb
    rv_allow = MOM * 3 * N.STAT_TERMS * N.EPS32 * ex2 * (M / (M - 1) if M > 1 else 1) + 4 * N.EPS32 * rv_ref.abs()
    rr = ((rv.double() - rv_ref).abs() / rv_allow).max().item()
    assert rr <= 1.0, 'running_var off by %.3g x its allowance' % rr
    c.note('running_var', rr)

    yref, mag, K = N.bn_y_direct(x, mean.t, invstd.t, gamma, beta, relu, res)
    c.check('y', y.t, yref, mag, K)
    if relu and res is None:
        mask_equal(y.t > 0, N.relu_mask(x, mean.t, invstd.t, gamma, beta), 'forward ReLU')
    if side:
        bits_equal(y16.t, y.t.bfloat16(), 'y16')
        bits_equal(dx16.t, dx.t.bfloat16(), 'dx16')

    if res is not None:
        mask = y.t > 0
        bits_equal(gm.t, torch.where(mask, dy, torch.zeros_like(dy)), 'gmasked')
    elif relu:
        mask = N.relu_mask(x, mean.t, invstd.t, gamma, beta)
    else:
        mask = None
    r = N.bn_bwd_ref(x, dy, mask, mean.t, invstd.t)
    c.check('dbeta', db.t, r['dbeta'], r['mb'], N.STAT_TERMS + 2)
    c.check('dgamma', dg.t, r['dgamma'], r['mg'], N.STAT_TERMS + 6)
    dxr, mag, K = N.bn_dx_ref(r, gamma, invstd.t, dg.t, db.t, M)
    c.check('dx', dx.t, dxr, mag, K)
    return c.res


# ------------------------------------------------------------------ tfb_bn_fwd_stats
STATS_VARIANTS = ('plain', 'residual', 'y16')


def bn_fwd_stats(c, C, HW, nb, variant, shift=3.0, seed=10):
    """tfb_bn_fwd_stats from fp64 sums. variant: plain, residual, y16 (all with ReLU) or pool (the squeeze-excite means: the
    grid kernel, or the flat one for C / 4 <= 128 and HW >= 1024)."""
    M = HW * nb
    x = c.rand((M, C), seed, 1.5, shift)
    gamma, beta = c.affine(C, seed + 1)
    stats = _stats_fp64(x)
    res = c.rand((M, C), seed + 2) if variant == 'residual' else None
    pool = variant == 'pool'
    y, mean, invstd = c.out((M, C)), c.out((C,)), c.out((C,))
    y16 = c.out((M, C), torch.bfloat16) if variant == 'y16' else None
    pooled = c.out((nb, C)) if pool else None
    rm, rv = torch.zeros(C, device=c.dev), torch.ones(C, device=c.dev)

    def pre():
        rm.zero_()
        rv.fill_(1.0)
        if pool:
            pooled.t.zero_()                          # accumulated: zero on entry

    def launch():
        c('tfb_bn_fwd_stats', x, y.t, M, C, gamma, beta, EPS, MOM, 1, rm, rv, mean.t, invstd.t, stats, y16 and y16.t, res,
          pooled and pooled.t, nb if pool else 0)
    c.twice(launch, [o for o in (y, mean, invstd, y16, pooled) if o is not None], pre)

    m_ref, is_ref = N.stats_from_sums(stats[:C], stats[C:], float(M), EPS)
    bits_equal(mean.t, m_ref, 'save_mean')
    ulps = ((invstd.t.double() - is_ref.double()).abs() / N.ulp32(is_ref)).max().item()
    assert ulps <= 1.0, 'save_invstd %.3g fp32 ulps from fp64(sums)' % ulps      # (fp64 contraction of s1/N - mean^2 on the device)
    yref, mag, K = N.bn_y_scsh(x, mean.t, invstd.t, gamma, beta, True, res)
    c.check('y (stats)', y.t, yref, mag, K)
    if res is None:
        sc = (gamma * invstd.t).double()
        sh = (-mean.t.double() * sc + beta.double()).float().double()
        mask_equal(y.t > 0, x.double() * sc + sh > 0, 'forward ReLU (stats)')
    if y16 is not None:
        bits_equal(y16.t, y.t.bfloat16(), 'y16 (stats)')
    if pool:
        flat = C // 4 <= 128 and HW >= 1024
        pref, pmag = N.pooled_ref(y.t, nb, HW, C)
        c.check('pooled (stats, %s)' % ('flat' if flat else 'grid'), pooled.t, pref, pmag, N.pool_terms(HW, C, flat))
    return c.res


# ------------------------------------------------------------------ tfb_bn_fwd with the pooled means
def bn_fwd_pool(c, C, HW, nb, shift=1.0, seed=20):
    """tfb_bn_fwd (+ReLU) with `pooled`: pre-filled with garbage, which the statistics kernel must clear."""
    M = HW * nb
    x = c.rand((M, C), seed, 2.0, shift)
    gamma, beta = c.affine(C, seed + 1)
    y, mean, invstd, pooled = c.out((M, C)), c.out((C,)), c.out((C,)), c.out((nb, C))

    def launch():
        c('tfb_bn_fwd', x, y.t, M, C, gamma, beta, EPS, MOM, 1, None, None, mean.t, invstd.t, c.ws, None, None, pooled.t, nb)
    c.twice(launch, [y, mean, invstd, pooled], lambda: pooled.t.fill_(3.0e30))
    N.check_stats(mean.t, invstd.t, x, EPS, 'stats (pool)')
    yref, mag, K = N.bn_y_direct(x, mean.t, invstd.t, gamma, beta, True)
    c.check('y (pool)', y.t, yref, mag, K)
    mask_equal(y.t > 0, N.relu_mask(x, mean.t, invstd.t, gamma, beta), 'forward ReLU (pool)')
    pref, pmag = N.pooled_ref(y.t, nb, HW, C)
    c.check('pooled (bn_fwd)', pooled.t, pref, pmag, N.pool_terms(HW, C, False))
    return c.res


# ------------------------------------------------------------------ tfb_bn_bwd_se
def bn_bwd_se(c, C, hw, nb, side=False, seed=30):
    """tfb_bn_bwd_se (ReLU recomputed): the gradient of the BatchNorm output is dy * gate[n] + dpool[n] / hw."""
    M = hw * nb
    x = c.rand((M, C), seed, 1.5, 0.5)
    gamma, beta = c.affine(C, seed + 1)
    mean, invstd = N.stats_from_sums(x.double().sum(0), (x.double() ** 2).sum(0), float(M), EPS)
    dy = c.rand((M, C), seed + 2)
    gate = torch.sigmoid(c.rand((nb, C), seed + 3))
    dpool = c.rand((nb, C), seed + 4, 4.0)
    dx, dg, db = c.out((M, C)), c.out((C,)), c.out((C,))
    dx16 = c.out((M, C), torch.bfloat16) if side else None

    def launch():
        c('tfb_bn_bwd_se', x, dy, dx.t, M, C, gamma, beta, mean, invstd, 1, dg.t, db.t, c.ws, dx16 and dx16.t, gate, dpool, hw)
    c.twice(launch, [o for o in (dx, dg, db, dx16) if o is not None])
    ga, dp = gate.double().repeat_interleave(hw, 0), dpool.double().repeat_interleave(hw, 0)
    g = dy.double() * ga + dp / hw
    gmag = (dy.double() * ga).abs() + dp.abs() / hw
    r = N.bn_bwd_ref(x, g, N.relu_mask(x, mean, invstd, gamma, beta), mean, invstd, gmag)
    c.check('dbeta (se)', db.t, r['dbeta'], r['mb'], N.STAT_TERMS + 4)
    c.check('dgamma (se)', dg.t, r['dgamma'], r['mg'], N.STAT_TERMS + 8)
    dxr, mag, K = N.bn_dx_ref(r, gamma, invstd, dg.t, db.t, M)
    c.check('dx (se)', dx.t, dxr, mag, K + 2)
    if side:
        bits_equal(dx16.t, dx.t.bfloat16(), 'dx16 (se)')
    return c.res


# ------------------------------------------------------------------ tfb_bn_apply (eval)
def bn_apply(c, C, M, variant, seed=40):
    """Eval-mode BatchNorm from running statistics. variant: relu, residual (relu(bn(x) + res)), y16 (relu + bf16 sidecar)."""
    x = c.rand((M, C), seed, 2.0, 0.3)
    gamma, beta = c.affine(C, seed + 1)
    mean = c.rand((C,), seed + 2, 0.5)
    invstd = (1.0 / torch.sqrt(c.rand((C,), seed + 3) ** 2 + 0.5)).float()
    res = c.rand((M, C), seed + 4) if variant == 'residual' else None
    y = c.out((M, C))
    y16 = c.out((M, C), torch.bfloat16) if variant == 'y16' else None

    def launch():
        c('tfb_bn_apply', x, y.t, M, C, gamma, beta, mean, invstd, 1, y16 and y16.t, res)
    c.twice(launch, [o for o in (y, y16) if o is not None])
    yref, mag, K = N.bn_y_direct(x, mean, invstd, gamma, beta, True, res)
    c.check('y (eval)', y.t, yref, mag, K)
    if res is None:
        mask_equal(y.t > 0, N.relu_mask(x, mean, invstd, gamma, beta), 'eval ReLU')
    if y16 is not None:
        bits_equal(y16.t, y.t.bfloat16(), 'y16 (eval)')
    return c.res


# ------------------------------------------------------------------ tfb_colsum
COLSUM_LAYOUTS = ('dense', 'padded', 'offset')


def colsum(c, C, M, layout, seed=50):
    """out[c] = sum over rows. dense: ldx == C; padded: ldx = C + 4 (and C + 3 when C % 4 != 0); offset: a column-offset view
    (4 bytes off 16-byte alignment: the scalar kernel)."""
    ld = {'dense': C, 'padded': C + (4 if C % 4 == 0 else 3), 'offset': C + 5}[layout]
    col = 1 if layout == 'offset' else 0
    full = c.rand((M, ld), seed, 1.0, 0.25)
    x = full[:, col:col + C]
    out = c.out((C,))
    c.twice(lambda: c('tfb_colsum', x, ld, M, C, out.t, c.ws), [out])
    xd = x.double()
    c.check('colsum', out.t, xd.sum(0), xd.abs().sum(0), N.STAT_TERMS + 2)
    return c.res


# ------------------------------------------------------------------ tfb_grad_prep
GRAD_PREP_OUTS = (('g32',), ('g16',), ('dbias',), ('g32', 'g16', 'dbias'))


def grad_prep(c, C, M, outs, relu, seed=60):
    """g = relu ? dy * (y > 0) : dy; g32 must be the masked dy bit for bit, g16 bf16(g) bit for bit, dbias the fp64 column sum of g
    at the fp32 partial length tfb_grad_prep uses (norm_ref.grad_prep_terms)."""
    dy = c.rand((M, C), seed, 1.0, 0.1)
    y = c.rand((M, C), seed + 1) if relu else None
    g32 = c.out((M, C)) if 'g32' in outs else None
    g16 = c.out((M, C), torch.bfloat16) if 'g16' in outs else None
    db = c.out((C,)) if 'dbias' in outs else None

    def launch():
        c('tfb_grad_prep', dy, y, g32 and g32.t, g16 and g16.t, db and db.t, c.ws if db is not None else None, M, C)
    c.twice(launch, [o for o in (g32, g16, db) if o is not None])
    g = torch.where(y > 0, dy, torch.zeros_like(dy)) if relu else dy
    if g32 is not None:
        bits_equal(g32.t, g, 'g32')
    if g16 is not None:
        bits_equal(g16.t, g.bfloat16(), 'g16')
    if db is not None:
        gd = g.double()
        c.check('dbias', db.t, gd.sum(0), gd.abs().sum(0), N.grad_prep_terms(M, C, c.sms))
    return c.res


# ------------------------------------------------------------------ LayerNorm
def layernorm(c, C, R, accumulate=False, seed=70):
    """tfb_layernorm_fwd (with the bf16 copy) then tfb_layernorm_bwd (dx overwritten, or accumulated onto given values)."""
    x = c.rand((R, C), seed, 1.3, 0.4)
    gamma, beta = c.affine(C, seed + 1)
    dy = c.rand((R, C), seed + 2)
    d0 = c.rand((R, C), seed + 3)
    y, y16, mean, rstd = c.out((R, C)), c.out((R, C), torch.bfloat16), c.out((R,)), c.out((R,))
    dx, dg, db = c.out((R, C)), c.out((C,)), c.out((C,))

    def launch():
        c('tfb_layernorm_fwd', x, y.t, R, C, gamma, beta, EPS, mean.t, rstd.t, y16.t)
        c('tfb_layernorm_bwd', x, dy, dx.t, R, C, gamma, mean.t, rstd.t, dg.t, db.t, int(accumulate), c.ws)
    c.twice(launch, [y, y16, mean, rstd, dx, dg, db], (lambda: dx.t.copy_(d0)) if accumulate else None)
    rm, rr = N.check_ln_stats(mean.t, rstd.t, x, EPS, 'LayerNorm C %d' % C)
    c.note('ln mean', rm)
    c.note('ln rstd', rr)
    yref, mag, K = N.ln_fwd_ref(x, mean.t, rstd.t, gamma, beta)
    c.check('ln y', y.t, yref, mag, K)
    bits_equal(y16.t, y.t.bfloat16(), 'ln y16')
    dxr, mag, K = N.ln_dx_ref(x, dy, gamma, mean.t, rstd.t)
    if accumulate:
        dxr, mag, K = dxr + d0.double(), mag + d0.double().abs(), K + 1
    c.check('ln dx', dx.t, dxr, mag, K)
    p = N.ln_param_ref(x, dy, mean.t, rstd.t)
    c.check('ln dbeta', db.t, p['dbeta'], p['mb'], N.ln_param_terms(R))
    c.check('ln dgamma', dg.t, p['dgamma'], p['mg'], N.ln_param_terms(R))
    return c.res


def add_dropout_ln(c, C, R, p, with_gx, seed=80):
    """tfb_add_dropout_ln_fwd / _bwd. xnew must be res + tfb_dropout(x) bit for bit, dx = dres * keep-scale bit for bit with the
    keep-scale taken from tfb_dropout applied to ones; h, dres and the parameter gradients against fp64 from the kernel's xnew and
    row statistics."""
    res, x = c.rand((R, C), seed), c.rand((R, C), seed + 1, 0.7)
    gamma, beta = c.affine(C, seed + 2)
    dh = c.rand((R, C), seed + 3)
    gx = c.rand((R, C), seed + 4, 0.5) if with_gx else None
    seed_dev = torch.tensor([SEED], dtype=torch.int64, device=c.dev)
    off = 977
    xnew, h, h16, mean, rstd = c.out((R, C)), c.out((R, C)), c.out((R, C), torch.bfloat16), c.out((R,)), c.out((R,))
    dres, dx, dg, db = c.out((R, C)), c.out((R, C)), c.out((C,)), c.out((C,))

    def launch():
        c('tfb_add_dropout_ln_fwd', res, x, xnew.t, h.t, R, C, gamma, beta, EPS, p, seed_dev, off, mean.t, rstd.t, h16.t)
        c('tfb_add_dropout_ln_bwd', xnew.t, dh, gx, dres.t, dx.t, R, C, gamma, mean.t, rstd.t, p, seed_dev, off, dg.t, db.t, c.ws)
    c.twice(launch, [xnew, h, h16, mean, rstd, dres, dx, dg, db])

    want = torch.empty_like(x)
    c('tfb_dropout', x, want, R * C, p, seed_dev, off, res)
    bits_equal(xnew.t, want, 'xnew')
    keep = torch.empty_like(x)
    c('tfb_dropout', torch.ones_like(x), keep, R * C, p, seed_dev, off, None)
    bits_equal(dx.t, dres.t * keep, 'dx = dres * keep')
    if p > 0:
        frac = (keep == 0).double().mean().item()
        assert abs(frac - p) < 5 * math.sqrt(p * (1 - p) / keep.numel()) + 1e-3, 'dropped fraction %.4f for p %g' % (frac, p)
    c.note('adln mean', N.check_ln_stats(mean.t, rstd.t, xnew.t, EPS, 'add_dropout_ln')[0])
    href, mag, K = N.ln_fwd_ref(xnew.t, mean.t, rstd.t, gamma, beta)
    c.check('adln h', h.t, href, mag, K)
    bits_equal(h16.t, h.t.bfloat16(), 'h16')
    dr, mag, K = N.ln_dx_ref(xnew.t, dh, gamma, mean.t, rstd.t)
    if gx is not None:
        dr, mag, K = dr + gx.double(), mag + gx.double().abs(), K + 1
    c.check('adln dres', dres.t, dr, mag, K)
    pr = N.ln_param_ref(xnew.t, dh, mean.t, rstd.t)
    c.check('adln dbeta', db.t, pr['dbeta'], pr['mb'], N.ln_param_terms(R))
    c.check('adln dgamma', dg.t, pr['dgamma'], pr['mg'], N.ln_param_terms(R))
    return c.res


# ------------------------------------------------------------------ one stream, many shapes
def stream_reuse(c, calls):
    """calls: [(case function, args)]. Each case alone, then all of them back to back on the same stream and workspace (the stream's
    scratch, partials and arrival counters shared): every output the same bits as alone."""
    def capture(fn, args):
        outs = []
        real = c.twice
        c.twice = lambda *a, **k: (real(*a, **k), outs.append(c.last))
        try:
            fn(c, *args)
        finally:
            c.twice = real
        return [b for o in outs for b in o]
    alone = [capture(fn, args) for fn, args in calls]
    together = [capture(fn, args) for fn, args in calls]
    for (fn, args), a, b in zip(calls, alone, together):
        assert len(a) == len(b) and all(torch.equal(u, v) for u, v in zip(a, b)), '%s%s differs in sequence' % (fn.__name__, args)


# ------------------------------------------------------------------ refusals (host-side, nothing is launched)
def refusals(c):
    """Operands the apply passes cannot access (4 bytes off 16-byte alignment, 2 bytes off the 8 of a bf16 sidecar) and C > 2048
    for the statistics-reading pass are refused with `argument check failed` before any launch."""
    M, C, nb = 8, 8, 2
    buf = torch.zeros(M * C + 8, device=c.dev)
    a, off = buf[:M * C], buf[1:1 + M * C]                     # off: a contiguous view 4 bytes past an aligned address
    b16 = torch.zeros(M * C + 8, dtype=torch.bfloat16, device=c.dev)
    h, hoff = b16[:M * C], b16[1:1 + M * C]
    v = lambda n=C: torch.ones(n, device=c.dev)
    voff = torch.ones(C + 4, device=c.dev)[1:1 + C]
    stats = torch.zeros(2 * C, dtype=torch.float64, device=c.dev)
    g = torch.ones(nb * C, device=c.dev)
    goff = torch.ones(nb * C + 4, device=c.dev)[1:1 + nb * C]
    sl = torch.zeros(2 * C + 1, dtype=torch.float64, device=c.dev)
    cnt = torch.tensor([float(M)], dtype=torch.float64, device=c.dev)

    def fwd(x=a, y=a, res=None, y16=None, gamma=None, mean=None):
        return ('tfb_bn_fwd', x, y, M, C, gamma if gamma is not None else v(), v(), EPS, MOM, 1, None, None,
                mean if mean is not None else v(), v(), c.ws, y16, res, None, 0)

    def fwd_stats(x=a, y=a, res=None, y16=None, CC=C):
        return ('tfb_bn_fwd_stats', x, y, M, CC, v(CC), v(CC), EPS, MOM, 1, None, None, v(CC), v(CC),
                torch.zeros(2 * CC, dtype=torch.float64, device=c.dev), y16, res, None, 0)

    def apply(x=a, y=a, res=None, y16=None, invstd=None):
        return ('tfb_bn_apply', x, y, M, C, v(), v(), v(), invstd if invstd is not None else v(), 1, y16, res)

    def bwd(x=a, dy=a, dx=a, dx16=None, ymask=None, gm=None):
        return ('tfb_bn_bwd', x, dy, dx, M, C, v(), v(), v(), v(), 0, v(), v(), c.ws, dx16, ymask, gm)

    def bwd_se(x=a, dy=a, dx=a, dx16=None, gate=g, dpool=g):
        return ('tfb_bn_bwd_se', x, dy, dx, M, C, v(), v(), v(), v(), 1, v(), v(), c.ws, dx16, gate, dpool, M // nb)

    def fwd_sync(x=a, y=a, res=None, y16=None, from_stats=0):
        return ('tfb_bn_fwd_sync', x, y, M, C, v(), v(), EPS, MOM, 1, None, None, v(), v(), sl, 1, sl.clone(), from_stats, y16, res, None, 0)

    def sync_reduce(x=a, dy=a, ymask=None, gate=None, dpool=None):
        return ('tfb_bn_bwd_sync_reduce', x, dy, M, C, v(), v(), v(), v(), 0, v(), v(), c.ws, ymask, gate, dpool, M // nb,
                torch.zeros(2 * C, dtype=torch.float64, device=c.dev))

    def sync_apply(x=a, dy=a, dx=a, dx16=None, ymask=None, gm=None, gate=None, dpool=None):
        return ('tfb_bn_bwd_sync_apply', x, dy, dx, M, C, v(), v(), v(), v(), 0, sl[:2 * C], 1, cnt, v(2 * C), dx16, ymask, gm, gate, dpool,
                M // nb)

    bad = {fwd: [dict(x=off), dict(y=off), dict(res=off), dict(y16=hoff), dict(gamma=voff), dict(mean=voff)],
           fwd_stats: [dict(x=off), dict(y=off), dict(res=off), dict(y16=hoff), dict(CC=2052)],
           apply: [dict(x=off), dict(y=off), dict(res=off), dict(y16=hoff), dict(invstd=voff)],
           bwd: [dict(x=off), dict(dy=off), dict(dx=off), dict(dx16=hoff), dict(ymask=off), dict(ymask=a, gm=off)],
           bwd_se: [dict(x=off), dict(dy=off), dict(dx=off), dict(dx16=hoff), dict(gate=goff), dict(dpool=goff)],
           fwd_sync: [dict(x=off), dict(y=off), dict(res=off), dict(y16=hoff), dict(x=off, from_stats=1)],
           sync_reduce: [dict(x=off), dict(dy=off), dict(ymask=off), dict(gate=goff, dpool=g), dict(gate=g, dpool=goff)],
           sync_apply: [dict(x=off), dict(dy=off), dict(dx=off), dict(dx16=hoff), dict(ymask=off), dict(ymask=a, gm=off),
                        dict(gate=goff, dpool=g), dict(gate=g, dpool=goff)]}
    for make, kws in bad.items():
        for kw in kws:
            with pytest.raises(RuntimeError, match='argument check failed'):
                c.call(*make(**kw))
        c(*make())                                          # the same call with aligned operands is accepted
