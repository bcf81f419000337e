"""Cases of the elementwise, upsample and squeeze-excite kernels (csrc/elementwise.cu), shared by tests/test_elementwise_exact.py
(H100, full sizes) and tests/test_elementwise_emulated.py (CPU emulation, reduced sizes that still cross every dispatch boundary).
Every case runs twice into NaN-filled, sentinel-guarded outputs (tc_ref.Guarded), and the two runs give the same bits. Outputs are
compared element by element with the float64 references of tests/elementwise_ref.py, or bit for bit where the kernel's result is
one fp32 (or bf16) rounding of its inputs that the reference can restate. A case returns {check: worst allowance ratio}."""
import pytest
import torch

import elementwise_ref as R
from tc_ref import Guarded, check

TOL = 1e-3                # relative L2: a backstop only, the element-wise allowance is the check


class Ctx:
    def __init__(self, call, dev, sms):
        self.call, self.dev, self.sms = call, dev, sms
        self.res = {}

    def rand(self, shape, seed, scale=1.0, shift=0.0):
        g = torch.Generator(device=self.dev).manual_seed(seed)
        return torch.randn(shape, generator=g, device=self.dev) * scale + shift

    def out(self, shape, dtype=torch.float32):
        return Guarded(shape, dtype, self.dev)

    def sync(self):
        if torch.device(self.dev).type == 'cuda':
            torch.cuda.synchronize()

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
        for i, (a, b) in enumerate(zip(*runs)):
            assert torch.equal(a, b), 'output %d differs between two launches' % i

    def check(self, name, out, ref, mag, K, slack=None):
        _, ratio = check(out, ref, mag, K, TOL, slack, name, floor=1e-3 * mag.double().norm().item())
        self.res[name] = max(self.res.get(name, 0.0), ratio)
        return ratio


def bits_equal(a, b, what):
    a, b = a.contiguous(), b.contiguous()
    view = torch.int16 if a.dtype == torch.bfloat16 else torch.int32
    ne = a.view(view) != b.view(view)
    assert not bool(ne.any()), '%s: %d elements differ, first at %s' % (what, int(ne.sum()), tuple(int(i) for i in ne.nonzero()[0]))


# ------------------------------------------------------------------ bilinear upsample
def upsample(c, N, Hi, Wi, Ho, Wo, C, ac, side=False, seed=0):
    """tfb_upsample_bilinear_fwd (+ the bf16 sidecar) and tfb_upsample_bilinear_bwd. C % 4 == 0 takes the float4 forms (the backward
    only for windows the host guard admits), C % 4 != 0 the scalar ones (the scalar gather loops over windows wider than
    GATHER_W)."""
    x = c.rand((N, Hi, Wi, C), seed)
    dy = c.rand((N, Ho, Wo, C), seed + 1)
    y, dx = c.out((N, Ho, Wo, C)), c.out((N, Hi, Wi, C))
    y16 = c.out((N, Ho, Wo, C), torch.bfloat16) if side else None

    def launch():
        c.call('tfb_upsample_bilinear_fwd', x, y.t, N, Hi, Wi, Ho, Wo, C, ac, y16 and y16.t)
        c.call('tfb_upsample_bilinear_bwd', dy, dx.t, N, Hi, Wi, Ho, Wo, C, ac)
    c.twice(launch, [o for o in (y, dx, y16) if o is not None])
    ref, mag, slack, K = R.upsample_fwd_ref(x, Ho, Wo, ac)
    c.check('upsample y', y.t, ref, mag, K, slack)
    if side:
        bits_equal(y16.t, y.t.bfloat16(), 'upsample y16')
    ref, mag, slack, K = R.upsample_bwd_ref(dy, Hi, Wi, ac)
    c.check('upsample dx', dx.t, ref, mag, K, slack)
    return c.res


def gpt_up_add(c, N, H, W, C, gh, gw, side=False, seed=10):
    """tfb_gpt_up_add_fwd (float4 when C % 4 == 0, scalar otherwise; bf16 sidecar) and tfb_gpt_up_add_bwd with the (C, gh, gw) view
    of a token slab that leaves untouched token rows on both sides: those rows must keep their NaNs."""
    G = gh * gw
    t_off = 3
    T = t_off + G + 5
    feat = c.rand((N, H, W, C), seed)
    tok = c.rand((N, T, C), seed + 1)
    dy = c.rand((N, H, W, C), seed + 2)
    out, dtok = c.out((N, H, W, C)), c.out((N, T, C))
    out16 = c.out((N, H, W, C), torch.bfloat16) if side else None

    def launch():
        c.call('tfb_gpt_up_add_fwd', feat, tok, out.t, N, H, W, C, gh, gw, t_off, T, out16 and out16.t)
        c.call('tfb_gpt_up_add_bwd', dy, dtok.t, N, H, W, C, gh, gw, t_off, T)
    c.twice(launch, [o for o in (out, dtok, out16) if o is not None])
    up, mag, slack, K = R.upsample_fwd_ref(R.slab_view(tok, t_off, gh, gw), H, W, 0)
    c.check('gpt_up_add out', out.t, feat.double() + up, feat.double().abs() + mag, K + 2, slack)
    if side:
        bits_equal(out16.t, out.t.bfloat16(), 'gpt_up_add out16')
    ref, mag, slack, K = R.upsample_bwd_ref(dy, gh, gw, 0)          # [N, gh, gw, C] in the slab's (C, gh, gw) view
    c.check('gpt_up_add dtok', R.slab_view(dtok.t, t_off, gh, gw), ref, mag, K, slack)
    assert torch.isnan(dtok.t[:, :t_off]).all() and torch.isnan(dtok.t[:, t_off + G:]).all(), 'token rows outside the slab written'
    return c.res


# ------------------------------------------------------------------ squeeze-excite and pooling
def pool_hw(c, N, HW, C, seed=20):
    """tfb_pool_hw_fwd (split counts 1 .. 32) and tfb_pool_hw_bwd, overwriting and accumulating."""
    x = c.rand((N, HW, C), seed, 1.0, 0.5)
    d = c.rand((N, C), seed + 1)
    base = c.rand((N, HW, C), seed + 2)
    out, dx, dxa = c.out((N, C)), c.out((N, HW, C)), c.out((N, HW, C))

    def launch():
        c.call('tfb_pool_hw_fwd', x, out.t, N, HW, C)
        c.call('tfb_pool_hw_bwd', d, dx.t, N, HW, C, 0)
        dxa.t.copy_(base)
        c.call('tfb_pool_hw_bwd', d, dxa.t, N, HW, C, 1)
    c.twice(launch, [out, dx, dxa])
    s = R.fp32_recip(HW)
    xd = x.double()
    c.check('pool_hw', out.t, xd.sum(1) * s, xd.abs().sum(1) * s, R.pool_terms(HW))
    v = (d * s).unsqueeze(1).expand(N, HW, C)                        # fp32 product: exact restatement
    bits_equal(dx.t, v, 'pool_hw_bwd')
    c.check('pool_hw_bwd acc', dxa.t, base.double() + v.double(), base.double().abs() + v.double().abs(), 2)
    return c.res


def se_reduce(c, N, HW, C, seed=30):
    """tfb_se_bwd_reduce: dgate[n][c] = sum over the pixels of x * dy, on the flat kernel (C / 4 <= 128, HW >= 1024) or the slab
    kernel."""
    x, dy = c.rand((N, HW, C), seed, 1.0, 0.3), c.rand((N, HW, C), seed + 1)
    dg = c.out((N, C))
    c.twice(lambda: c.call('tfb_se_bwd_reduce', x, dy, dg.t, N, HW, C), [dg])
    p = x.double() * dy.double()
    c.check('se_reduce (%s)' % ('flat' if R.se_reduce_flat(HW, C) else 'slab'), dg.t, p.sum(1), p.abs().sum(1),
            R.se_reduce_terms(N, HW, C, c.sms))
    return c.res


def se_scale(c, N, HW, C, side=False, seed=40):
    """tfb_se_scale_fwd (one fp32 product: bit for bit; the bf16 sidecar bit for bit) and tfb_se_bwd_apply (fmaf(dpool, 1 / HW,
    dy * gate): two roundings), VEC 4 when C % 4 == 0 and VEC 1 otherwise."""
    x, dy = c.rand((N, HW, C), seed), c.rand((N, HW, C), seed + 1)
    gate = torch.sigmoid(c.rand((N, C), seed + 2))
    dpool = c.rand((N, C), seed + 3, 3.0)
    y, dx = c.out((N, HW, C)), c.out((N, HW, C))
    y16 = c.out((N, HW, C), torch.bfloat16) if side else None

    def launch():
        c.call('tfb_se_scale_fwd', x, gate, y.t, N, HW, C, y16 and y16.t)
        c.call('tfb_se_bwd_apply', dy, gate, dpool, dx.t, N, HW, C)
    c.twice(launch, [o for o in (y, dx, y16) if o is not None])
    bits_equal(y.t, x * gate.unsqueeze(1), 'se_scale y')
    if side:
        bits_equal(y16.t, y.t.bfloat16(), 'se_scale y16')
    s = R.fp32_recip(HW)
    a = (dy * gate.unsqueeze(1)).double()                              # the fp32 product, then the fma
    b = (dpool.double() * s).unsqueeze(1)
    c.check('se_bwd_apply', dx.t, a + b, a.abs() + b.abs(), 2)
    return c.res


def se_mlp_bwd(c, N, C, Cr, seed=50):
    """tfb_se_mlp_bwd: dw1, db1, dw2, db2 and dpool against the fp64 chain, with h holding negatives (the ReLU mask)."""
    dgate, gate = c.rand((N, C), seed), torch.sigmoid(c.rand((N, C), seed + 1))
    h = torch.relu(c.rand((N, Cr), seed + 2, 1.0, 0.2))
    pooled = c.rand((N, C), seed + 3)
    w1, w2 = c.rand((Cr, C), seed + 4, 0.2), c.rand((C, Cr), seed + 5, 0.2)
    dw1, db1, dw2, db2, dpool = c.out((Cr, C)), c.out((Cr,)), c.out((C, Cr)), c.out((C,)), c.out((N, C))
    part = torch.zeros(1, device=c.dev)
    c.twice(lambda: c.call('tfb_se_mlp_bwd', dgate, gate, h, pooled, w1, w2, dw1.t, db1.t, dw2.t, db2.t, dpool.t, part, N, C, Cr),
            [dw1, db1, dw2, db2, dpool])
    ref = R.se_mlp_bwd_ref(dgate, gate, h, pooled, w1, w2)
    for name, o in (('db2', db2), ('dw2', dw2), ('db1', db1), ('dw1', dw1), ('dpool', dpool)):
        r, mag, K = ref[name]
        c.check('se_mlp ' + name, o.t, r, mag, K)
    return c.res


# ------------------------------------------------------------------ token build (p_drop = 0)
def tokens(c, N, C, img_hw, img_grid, lid_hw, lid_grid, seed=60):
    """tfb_tokens_fwd and tfb_tokens_bwd (accumulate_feat 0 and 1) at p_drop = 0; dpos is the sum of g over the samples."""
    (Hi, Wi), (ghi, gwi), (Hl, Wl), (ghl, gwl) = img_hw, img_grid, lid_hw, lid_grid
    T = ghi * gwi + ghl * gwl
    img, lid = c.rand((N, Hi, Wi, C), seed), c.rand((N, Hl, Wl, C), seed + 1)
    pos = c.rand((T, C), seed + 2, 0.1)
    g = c.rand((N, T, C), seed + 3)
    bi, bl = c.rand((N, Hi, Wi, C), seed + 4), c.rand((N, Hl, Wl, C), seed + 5)
    seed_dev = torch.zeros(1, dtype=torch.int64, device=c.dev)
    tok, di, dl, dpos = c.out((N, T, C)), c.out((N, Hi, Wi, C)), c.out((N, Hl, Wl, C)), c.out((T, C))
    dia, dla, dposa = c.out((N, Hi, Wi, C)), c.out((N, Hl, Wl, C)), c.out((T, C))

    def launch():
        c.call('tfb_tokens_fwd', img, Hi, Wi, ghi, gwi, lid, Hl, Wl, ghl, gwl, pos, tok.t, N, C, 0.0, seed_dev, 5)
        c.call('tfb_tokens_bwd', g, di.t, Hi, Wi, ghi, gwi, dl.t, Hl, Wl, ghl, gwl, dpos.t, N, C, 0.0, seed_dev, 5, 0)
        dia.t.copy_(bi)
        dla.t.copy_(bl)
        c.call('tfb_tokens_bwd', g, dia.t, Hi, Wi, ghi, gwi, dla.t, Hl, Wl, ghl, gwl, dposa.t, N, C, 0.0, seed_dev, 5, 1)
    c.twice(launch, [tok, di, dl, dpos, dia, dla, dposa])

    def pool(x, H, W, gh, gw):
        wh, ww = H // gh, W // gw
        v = x.double().view(N, gh, wh, gw, ww, C)
        return v.sum((2, 4)).reshape(N, gh * gw, C), v.abs().sum((2, 4)).reshape(N, gh * gw, C), wh * ww
    si, mi, ki = pool(img, Hi, Wi, ghi, gwi)
    sl, ml, kl = pool(lid, Hl, Wl, ghl, gwl)
    # each token: a sequential fp32 sum of its window, the division by wh * ww, the add of pos
    ref = pos.double() + torch.cat([si / ki, sl / kl], 1)
    mag = pos.double().abs() + torch.cat([mi / ki, ml / kl], 1)
    c.check('tokens', tok.t, ref, mag, max(ki, kl) + 2)

    def spread(gt, H, W, gh, gw):
        wh, ww = H // gh, W // gw
        v = gt * R.fp32_recip(wh * ww)                                 # fp32 product: the kernel's g * 1 * inv
        v = v.view(N, gh, 1, gw, 1, C).expand(N, gh, wh, gw, ww, C)
        return v.reshape(N, H, W, C)
    gi, gl = spread(g[:, :ghi * gwi], Hi, Wi, ghi, gwi), spread(g[:, ghi * gwi:], Hl, Wl, ghl, gwl)
    bits_equal(di.t, gi, 'tokens dimg')
    bits_equal(dl.t, gl, 'tokens dlid')
    c.check('tokens dimg acc', dia.t, bi.double() + gi.double(), bi.double().abs() + gi.double().abs(), 2)
    c.check('tokens dlid acc', dla.t, bl.double() + gl.double(), bl.double().abs() + gl.double().abs(), 2)
    gd = g.double()
    c.check('tokens dpos', dpos.t, gd.sum(0), gd.abs().sum(0), N)
    bits_equal(dposa.t, dpos.t, 'tokens dpos (accumulate_feat)')
    return c.res


def transpose(c, N, A, B, seed=70):
    """tfb_transpose_last2: a permutation, bit for bit."""
    x = c.rand((N, A, B), seed)
    y = c.out((N, B, A))
    c.twice(lambda: c.call('tfb_transpose_last2', x, y.t, N, A, B), [y])
    bits_equal(y.t, x.transpose(1, 2), 'transpose_last2')
    return c.res


def image_prep(c, N, H, W, seed=80):
    """tfb_image_prep: ((x / 255) - mean) / std in fp32 (two correctly rounded divisions and a subtraction), bit for bit, NCHW ->
    NHWC. Each step is restated in fp64 from fp32 operands and rounded to fp32, which is the correctly rounded fp32 result (53 >= 2 * 24
    + 2 bits: the double rounding is harmless); torch's own fp32 division by a scalar multiplies by the reciprocal on some devices."""
    g = torch.Generator(device=c.dev).manual_seed(seed)
    img = torch.randint(0, 256, (N, 3, H, W), generator=g, device=c.dev).float()
    out = c.out((N, H, W, 3))
    c.twice(lambda: c.call('tfb_image_prep', img, out.t, N, H, W), [out])
    mean = torch.tensor([0.485, 0.456, 0.406], dtype=torch.float32, device=c.dev).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225], dtype=torch.float32, device=c.dev).view(1, 3, 1, 1)
    q = (img.double() / 255.0).float()
    q = (q.double() - mean.double()).float()
    q = (q.double() / std.double()).float()
    bits_equal(out.t, q.permute(0, 2, 3, 1), 'image_prep')
    return c.res


# ------------------------------------------------------------------ pointwise
def add_relu(c, n, relu, side, seed=90):
    """tfb_add_relu: one fp32 add (+ ReLU), bit for bit, n not a multiple of 4 (the scalar tail), with the bf16 sidecar."""
    a, b = c.rand((n,), seed), c.rand((n,), seed + 1)
    y = c.out((n,))
    y16 = c.out((n,), torch.bfloat16) if side else None
    c.twice(lambda: c.call('tfb_add_relu', a, b, y.t, n, int(relu), y16 and y16.t), [o for o in (y, y16) if o is not None])
    s = a + b
    bits_equal(y.t, torch.where(s > 0, s, torch.zeros_like(s)) if relu else s, 'add_relu')
    if side:
        bits_equal(y16.t, y.t.bfloat16(), 'add_relu y16')
    return c.res


def activations(c, n, seed=100):
    """tfb_relu_bwd (the mask exact: bit for bit), tfb_sigmoid_fwd over |x| up to 120 (expf overflows past 88) and tfb_sigmoid_bwd
    (three fp32 roundings)."""
    x = c.rand((n,), seed, 3.0)
    x[: min(n, 12)] = torch.tensor([0.0, -0.0, 88.0, -88.0, 88.8, -88.8, 89.0, -89.0, 104.0, -104.0, 120.0, -120.0],
                                   device=c.dev)[: min(n, 12)]
    dy = c.rand((n,), seed + 1)
    yv = torch.sigmoid(c.rand((n,), seed + 2, 2.0))
    dr, sg, ds = c.out((n,)), c.out((n,)), c.out((n,))

    def launch():
        c.call('tfb_relu_bwd', x, dy, dr.t, n)
        c.call('tfb_sigmoid_fwd', x, sg.t, n)
        c.call('tfb_sigmoid_bwd', yv, dy, ds.t, n)
    c.twice(launch, [dr, sg, ds])
    bits_equal(dr.t, torch.where(x > 0, dy, torch.zeros_like(dy)), 'relu_bwd')
    ref, mag, K = R.sigmoid_ref(x)
    c.check('sigmoid', sg.t, ref, mag, K)
    p = dy.double() * yv.double() * (1 - yv.double())
    c.check('sigmoid_bwd', ds.t, p, p.abs(), 3)
    return c.res


def stride2(c, N, H, W, C, seed=110):
    """tfb_subsample2 (with the bf16 sidecar) and tfb_dilate2 to fp32 and to bf16 (float4 form when C % 4 == 0): bit for bit."""
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    x, s = c.rand((N, H, W, C), seed), c.rand((N, Ho, Wo, C), seed + 1)
    xs, xs16 = c.out((N, Ho, Wo, C)), c.out((N, Ho, Wo, C), torch.bfloat16)
    d32, d16 = c.out((N, H, W, C)), c.out((N, H, W, C), torch.bfloat16)

    def launch():
        c.call('tfb_subsample2', x, xs.t, N, H, W, C, xs16.t)
        c.call('tfb_dilate2', s, d32.t, N, H, W, C, 0)
        c.call('tfb_dilate2', s, d16.t, N, H, W, C, 1)
    c.twice(launch, [xs, xs16, d32, d16])
    bits_equal(xs.t, x[:, ::2, ::2], 'subsample2')
    bits_equal(xs16.t, x[:, ::2, ::2].bfloat16(), 'subsample2 bf16')
    want = torch.zeros((N, H, W, C), device=c.dev)
    want[:, ::2, ::2] = s
    bits_equal(d32.t, want, 'dilate2')
    bits_equal(d16.t, want.bfloat16(), 'dilate2 bf16')
    return c.res


def scale_bcast(c, N, T, C, seed=120):
    """tfb_scale_dev (device scalar and none; overwrite: one product of fl32(s * k), bit for bit; accumulate: one fma) and
    tfb_bcast_add_nc (one add, bit for bit)."""
    n = N * T * C
    x, y0 = c.rand((n,), seed), c.rand((n,), seed + 1)
    s = c.rand((1,), seed + 2)
    k = 0.37
    v = c.rand((N, C), seed + 3)
    ya, yb, yacc, yb2 = c.out((n,)), c.out((n,)), c.out((n,)), c.out((N, T, C))

    def launch():
        c.call('tfb_scale_dev', x, s, k, ya.t, n, 0)
        c.call('tfb_scale_dev', x, None, k, yb.t, n, 0)
        yacc.t.copy_(y0)
        c.call('tfb_scale_dev', x, s, k, yacc.t, n, 1)
        c.call('tfb_bcast_add_nc', x.view(N, T, C), v, yb2.t, N, T, C)
    c.twice(launch, [ya, yb, yacc, yb2])
    f = s * R.f32(k).to(c.dev)
    bits_equal(ya.t, x * f, 'scale_dev')
    bits_equal(yb.t, x * R.f32(k).to(c.dev), 'scale_dev (no scalar)')
    p = x.double() * f.double()
    c.check('scale_dev acc', yacc.t, p + y0.double(), p.abs() + y0.double().abs(), 2)
    bits_equal(yb2.t, x.view(N, T, C) + v.unsqueeze(1), 'bcast_add_nc')
    return c.res


def softmax(c, rows, L, seed=130):
    """tfb_softmax_fwd (P and Pd separate, and Pd aliasing P) and tfb_softmax_bwd at p_drop = 0."""
    scale = 0.1443                                    # about 1 / sqrt(48), not a power of two
    S = c.rand((rows, L), seed, 6.0)
    dPd = c.rand((rows, L), seed + 1)
    seed_dev = torch.zeros(1, dtype=torch.int64, device=c.dev)
    P, Pd, Pa, dS = c.out((rows, L)), c.out((rows, L)), c.out((rows, L)), c.out((rows, L))

    def launch():
        c.call('tfb_softmax_fwd', S, P.t, Pd.t, rows, L, scale, 0.0, seed_dev, 3)
        c.call('tfb_softmax_fwd', S, Pa.t, Pa.t, rows, L, scale, 0.0, seed_dev, 3)
        c.call('tfb_softmax_bwd', P.t, dPd, dS.t, rows, L, scale, 0.0, seed_dev, 3)
    c.twice(launch, [P, Pd, Pa, dS])
    ref, mag, slack, K = R.softmax_ref(S, scale)
    c.check('softmax', P.t, ref, mag, K, slack)
    bits_equal(Pd.t, P.t, 'softmax Pd (p = 0)')
    bits_equal(Pa.t, P.t, 'softmax in place')
    ref, mag, K = R.softmax_bwd_ref(P.t, dPd, scale)
    c.check('softmax_bwd', dS.t, ref, mag, K)
    return c.res


# ------------------------------------------------------------------ misaligned operands (host side: refused, or the scalar form)
def misaligned(c, fallbacks=True):
    """Operands 4 bytes off 16-byte alignment (2 bytes off the 8 of a bf16 sidecar): the float4-only entry points refuse them with
    `argument check failed` before any launch. fallbacks: tfb_se_scale_fwd and tfb_se_bwd_apply take their scalar form and give the
    bits of the aligned call."""
    N, HW, C = 2, 5, 8
    n = N * HW * C
    buf = c.rand((n + 8,), 1)
    a, off = buf[:n].clone(), buf[1:1 + n]
    b16 = torch.zeros(n + 8, dtype=torch.bfloat16, device=c.dev)
    h, hoff = b16[:n], b16[1:1 + n]
    y = torch.zeros(n, device=c.dev)
    yoff = torch.zeros(n + 4, device=c.dev)[1:1 + n]
    nc = torch.ones(N * C, device=c.dev)
    ncoff = torch.ones(N * C + 4, device=c.dev)[1:1 + N * C]
    sd = torch.zeros(1, dtype=torch.int64, device=c.dev)

    refused = {
        'tfb_add_relu': lambda x=a, b=a, o=y, o16=None: (x, b, o, n, 1, o16),
        'tfb_dropout': lambda x=a, o=y, r=None: (x, o, n, 0.0, sd, 0, r),
        'tfb_cast_bf16': lambda x=a, o=h: (x, o, n),
        'tfb_pool_hw_fwd': lambda x=a: (x, torch.zeros(N * C, device=c.dev), N, HW, C),
        'tfb_se_bwd_reduce': lambda x=a, d=a: (x, d, torch.zeros(N * C, device=c.dev), N, HW, C),
    }
    bad = {'tfb_add_relu': [dict(x=off), dict(b=off), dict(o=yoff), dict(o16=hoff)],
           'tfb_dropout': [dict(x=off), dict(o=yoff), dict(r=off)],
           'tfb_cast_bf16': [dict(x=off), dict(o=hoff)],
           'tfb_pool_hw_fwd': [dict(x=off)],
           'tfb_se_bwd_reduce': [dict(x=off), dict(d=off)]}
    for name, kws in bad.items():
        for kw in kws:
            with pytest.raises(RuntimeError, match='argument check failed'):
                c.call(name, *refused[name](**kw))
        c.call(name, *refused[name]())                        # the same call with aligned operands is accepted
    c.sync()
    if not fallbacks:
        return

    gate = torch.sigmoid(c.rand((N * C,), 2))
    gbuf = torch.zeros(N * C + 4, device=c.dev)
    goff = gbuf[1:1 + N * C]
    goff.copy_(gate)
    dp = c.rand((N * C,), 3)
    dpbuf = torch.zeros(N * C + 4, device=c.dev)
    dpoff = dpbuf[1:1 + N * C]
    dpoff.copy_(dp)
    want_y, want_16, want_dx = torch.zeros(n, device=c.dev), torch.zeros(n, dtype=torch.bfloat16, device=c.dev), torch.zeros(n, device=c.dev)
    c.call('tfb_se_scale_fwd', a, gate, want_y, N, HW, C, want_16)
    c.call('tfb_se_bwd_apply', a, gate, dp, want_dx, N, HW, C)
    x_off = off
    x_off.copy_(a)
    for args in ((x_off, gate, yoff, None), (a, goff, y, None), (a, gate, y, hoff)):
        yoff.zero_(), y.zero_(), hoff.zero_()
        c.call('tfb_se_scale_fwd', args[0], args[1], args[2], N, HW, C, args[3])
        c.sync()
        bits_equal(args[2], want_y, 'se_scale_fwd (misaligned operand)')
        if args[3] is not None:
            bits_equal(args[3], want_16, 'se_scale_fwd y16 (misaligned)')
    for args in ((x_off, gate, dp, y), (a, goff, dp, y), (a, gate, dpoff, y), (a, gate, dp, yoff)):
        y.zero_(), yoff.zero_()
        c.call('tfb_se_bwd_apply', args[0], args[1], args[2], args[3], N, HW, C)
        c.sync()
        bits_equal(args[3], want_dx, 'se_bwd_apply (misaligned operand)')
