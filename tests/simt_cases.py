"""Cases of the exact-fp32 CUDA-core kernels (csrc/conv_simt.cu: tfb_conv2d_fwd / _dgrad / _wgrad; csrc/gemm_simt.cu:
tfb_gemm_f32_simt, tfb_gemm_small_m), shared by tests/test_simt_exact.py (H100, full sizes and the shapes of every call in a
benchmark step) and tests/test_simt_emulated.py (CPU emulation, reduced sizes that still cross every dispatch boundary).
Every case:
- runs twice into NaN-filled, sentinel-guarded outputs (tc_ref.Guarded) and the two runs give the same bits; dw / dbias start as
  NaN, so the launcher's clearing (or the stem's assigning fold) is part of what is checked;
- with kind 'exact' (dyadic operands, simt_ref.assert_exact) must equal the float64 result bit for bit, except through a sigmoid;
- with kind 'gauss' / 'shift' (Gaussian, and mean-shifted so that sums cancel) must stay within K * 2^-23 * (|a| |b|) per element,
  plus 2^-23 * |v| per epilogue rounding, and within relative L2 1e-3.
Operand buffers of the GEMMs are NaN wherever no operand element lies (leading-dimension gaps, batch gaps), and the output gaps must
still be NaN afterwards. A case returns {check: worst allowance ratio} for the caller to print."""
import math

import pytest
import torch

import simt_ref as R
from tc_ref import Guarded, check as tc_check

TOL = 1e-3                # relative L2: a backstop only, the element-wise allowance is the check
KINDS = ('exact', 'gauss', 'shift')


class Ctx:
    def __init__(self, call, dev, sms):
        self.call, self.dev, self.sms = call, dev, sms
        self.res = {}

    def out(self, shape):
        return Guarded(shape, torch.float32, self.dev)

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
        _, ratio = tc_check(out, ref, mag, K, TOL, slack, name, floor=1e-3 * mag.double().norm().item())
        self.res[name] = max(self.res.get(name, 0.0), ratio)
        return ratio

    def exact(self, name, out, ref):
        R.bits_equal(out, ref, name)
        self.res[name + ' (exact)'] = 0.0


# ------------------------------------------------------------------ convolutions
CONV_OPS = ('fwd', 'dgrad', 'wgrad')


def conv(c, N, H, W, Cin, Cout, k, stride, groups, bias, relu, kind, ops=CONV_OPS, seed=0):
    """tfb_conv2d_fwd (bias / relu as given), tfb_conv2d_dgrad and tfb_conv2d_wgrad (dbias when `bias`) of one shape."""
    dev = c.dev
    Ho, Wo = R.out_hw(H, W, k, stride)
    Cig, Cog, T = Cin // groups, Cout // groups, k * k
    npix = N * Ho * Wo
    if kind == 'exact':
        # x = i / 8, dy = i / 8 (|i| <= r, r narrowed for long wgrad contractions), w = j / 16 (|j| <= 8), bias = i / 128 (|i| <= 64)
        r = R.exact_range(npix)
        x, dy = R.dyadic((N, H, W, Cin), r, 3, seed, dev), R.dyadic((N, Ho, Wo, Cout), r, 3, seed + 3, dev)
        w = R.dyadic((Cout, Cig, k, k), 8, 4, seed + 1, dev)
        b = R.dyadic((Cout,), 64, 7, seed + 2, dev) if bias else None
        R.assert_exact(Cig * T, r / 8, 0.5, 2.0 ** -7, 0.5 if bias else 0.0, 'conv forward')
        R.assert_exact(Cog * T, r / 8, 0.5, 2.0 ** -7, 0.0, 'conv dgrad')
        R.assert_exact(npix, r / 8, r / 8, 2.0 ** -6, 0.0, 'conv wgrad')
    else:
        sh = 2.0 if kind == 'shift' else 0.0
        x, dy = R.gauss((N, H, W, Cin), seed, dev, 1.0, sh), R.gauss((N, Ho, Wo, Cout), seed + 3, dev, 1.0, sh * 0.75)
        w = R.gauss((Cout, Cig, k, k), seed + 1, dev, 1.0 / math.sqrt(Cig * T))
        b = R.gauss((Cout,), seed + 2, dev, 0.5) if bias else None
    args = (N, H, W, Cin, Cout, k, stride, groups)
    tag = ' %s' % kind
    if 'fwd' in ops:
        y = c.out((N, Ho, Wo, Cout))
        c.twice(lambda: c.call('tfb_conv2d_fwd', x, w, b, y.t, *args, int(relu)), [y])
        ref, mag = R.conv_fwd(x, w, b, stride, groups, relu)
        if kind == 'exact':
            c.exact('conv y', y.t, ref)
        else:
            c.check('conv y' + tag, y.t, ref, mag, Cig * T + 1)
    if 'dgrad' in ops:
        dx = c.out((N, H, W, Cin))
        c.twice(lambda: c.call('tfb_conv2d_dgrad', dy, w, dx.t, *args), [dx])
        ref, mag = R.conv_dgrad(dy, w, (N, H, W, Cin), stride, groups)
        if kind == 'exact':
            c.exact('conv dx', dx.t, ref)
        else:
            c.check('conv dx' + tag, dx.t, ref, mag, Cog * T)
    if 'wgrad' in ops:
        dw = c.out((Cout, Cig, k, k))
        db = c.out((Cout,)) if bias else None
        c.twice(lambda: c.call('tfb_conv2d_wgrad', x, dy, dw.t, db and db.t, *args), [o for o in (dw, db) if o is not None])
        ref, mag, dbr, dbm = R.conv_wgrad(x, dy, dw.t.shape, stride, groups)
        if kind == 'exact':
            c.exact('conv dw', dw.t, ref)
            if bias:
                c.exact('conv dbias', db.t, dbr)
        else:
            c.check('conv dw' + tag, dw.t, ref, mag, npix)
            if bias:
                c.check('conv dbias' + tag, db.t, dbr, dbm, npix)
    return c.res


def wgrad_path(N, H, W, Cin, Cout, k, stride, groups, sms):
    """(kernel, pixel splits, fused fold) that tfb_conv2d_wgrad picks for a shape on `sms` SMs (the launcher's arithmetic)."""
    Ho, Wo = R.out_hw(H, W, k, stride)
    npix = N * Ho * Wo
    cdiv = lambda a, b: -(-a // b)
    Cig, Cog = Cin // groups, Cout // groups
    ndw = Cout * Cig * k * k
    if groups == 1 and k == 1 and stride == 1 and Cout <= 16:
        cb = cdiv(Cin, 64)
        pp = cdiv(max(cdiv(npix, cdiv(4 * sms, cb)), 128), 16) * 16
        kern = 'narrowout'
    elif groups == 1 and Cin <= 4 and k == 3:
        cb = cdiv(Cout, 32)
        pp = cdiv(max(cdiv(npix, cdiv(4 * sms, cb)), 256), 8) * 8
        kern = 'smallcin'
    else:
        by = groups * cdiv(Cog, 32) * cdiv(Cig, 32)
        pp = cdiv(max(cdiv(npix, cdiv(4 * sms, by)), 256), 32) * 32
        kern = 'generic'
    return kern, cdiv(npix, pp), ndw <= 16384


# ------------------------------------------------------------------ tfb_gemm_f32_simt
def _layout(rows, cols, ld, nb, so, si, off):
    """(shape, strides, storage offset) of a [bo, bi, rows, cols] operand view and the buffer length it needs."""
    bo, bi = nb
    shape, strides = (bo, bi, rows, cols), (so, si, ld, 1)
    n = off + (bo - 1) * so + (bi - 1) * si + (rows - 1) * ld + cols if rows and cols else off + 1
    return shape, strides, off, max(n, 1)


def _operand(lay, kind, rng, e, seed, dev):
    """A NaN-filled buffer with operand values at every element the view covers."""
    shape, strides, off, n = lay
    buf = torch.full((n,), float('nan'), device=dev)
    if shape[2] and shape[3]:
        vals = R.dyadic(shape, rng, e, seed, dev) if kind == 'exact' else \
            R.gauss(shape, seed, dev, 1.0, 1.5 if kind == 'shift' else 0.0)
        for i in range(shape[0]):
            for j in range(shape[1]):
                buf.as_strided(shape[2:], strides[2:], off + i * strides[0] + j * strides[1]).copy_(vals[i, j])
    return buf


def _view(buf, lay):
    shape, strides, off, _ = lay
    return buf.as_strided(shape, strides, off)


def _moved(buf, lay, by):
    """The same values `by` floats further on (another alignment class of the same operand)."""
    b2 = torch.full((buf.numel() + by,), float('nan'), device=buf.device)
    b2[by:] = buf
    shape, strides, off, n = lay
    return b2, (shape, strides, off + by, n + by)


def _dyadic_scalar(v):
    return v == 0 or (math.frexp(abs(v))[0] == 0.5)


def gemm(c, ta, tb, M, N, K, kind, alpha=1.0, beta=0.0, bias=False, relu=False, lda=None, ldb=None, ldc=None, batch=(1, 1),
         strides=None, offs=(0, 0), seed=0):
    """C = alpha op(A) op(B) (+ bias) (+ beta C) (ReLU) over a two-level batch. strides: (sAo, sAi, sBo, sBi, sCo, sCi), default
    packed. offs: A / B storage offsets in floats (2: 8-byte but not 16-byte aligned; odd: the scalar loads). When every operand
    address is even the call takes the 8-byte loads: it is repeated with both operands one float further on (the scalar loads,
    the same values) and must give the same bits."""
    dev = c.dev
    ra, ca = (K, M) if ta else (M, K)
    rb, cb = (N, K) if tb else (K, N)
    lda, ldb, ldc = lda or ca, ldb or cb, ldc or N
    bo, bi = batch
    if strides is None:
        sAi, sBi, sCi = ra * lda, rb * ldb, M * ldc
        strides = (bi * sAi, sAi, bi * sBi, sBi, bi * sCi, sCi)
    sAo, sAi, sBo, sBi, sCo, sCi = strides
    if kind == 'exact':
        r = R.exact_range(K)
        assert _dyadic_scalar(alpha) and _dyadic_scalar(beta), 'exact operands need power-of-two alpha / beta'
        ea, eb = 3, 4                                          # A = i / 8, B = j / 16, bias = i / 128, C = i / 32
        grid = 2.0 ** -7 * min(1.0, abs(alpha) or 1.0, abs(beta) if beta else 1.0)
        R.assert_exact(K, abs(alpha) * r / 8, r / 16, grid, (0.5 if bias else 0.0) + abs(beta) * 1.0, 'gemm')
    else:
        r, ea, eb = 0, 0, 0
    la = _layout(ra, ca, lda, batch, sAo, sAi, offs[0])
    lb = _layout(rb, cb, ldb, batch, sBo, sBi, offs[1])
    lc = _layout(M, N, ldc, batch, sCo, sCi, 0)
    A = _operand(la, kind, r, ea, seed, dev)
    B = _operand(lb, kind, r, eb, seed + 1, dev)
    b = (R.dyadic((N,), 64, 7, seed + 2, dev) if kind == 'exact' else R.gauss((N,), seed + 2, dev, 0.5)) if bias else None
    C0 = R.dyadic((bo, bi, M, N), 32, 5, seed + 3, dev) if kind == 'exact' else R.gauss((bo, bi, M, N), seed + 3, dev)
    out = c.out((lc[3],))

    def pre():
        if beta != 0:
            _view(out.t, lc).copy_(C0)

    def launch(A=A, la=la, B=B, lb=lb):
        c.call('tfb_gemm_f32_simt', int(ta), int(tb), M, N, K, A[la[2]:], lda, B[lb[2]:], ldb, out.t, ldc, b, int(relu), float(alpha),
               float(beta), bo, bi, sAo, sAi, sBo, sBi, sCo, sCi)
    c.twice(launch, [out], pre)
    got = _view(out.t, lc)
    tag = 'gemm %s%s' % ('NT'[ta], 'NT'[tb])
    ref, mag = R.gemm(_view(A, la), _view(B, lb), ta, tb, alpha, beta, C0, b, relu)
    if kind == 'exact':
        c.exact(tag, got, ref)
    else:
        c.check('%s %s' % (tag, kind), got, ref, mag, K + 3)
    # the output gaps (ldc > N, batch gaps) are never written
    cover = torch.zeros(lc[3], dtype=torch.bool, device=dev)
    for i in range(bo):
        for j in range(bi):
            cover.as_strided((M, N), (ldc, 1), i * sCo + j * sCi).fill_(True)
    assert bool(out.t[~cover].isnan().all()), '%s wrote outside its output windows' % tag
    vec = all(v % 2 == 0 for v in (offs[0], offs[1], lda, ldb, sAo, sAi, sBo, sBi))
    if vec and M and N:
        first = out.bits()
        A1, la1 = _moved(A, la, 1)
        B1, lb1 = _moved(B, lb, 1)
        c.twice(lambda: launch(A1, la1, B1, lb1), [out], pre)
        assert torch.equal(out.bits(), first), '%s: the scalar loads give other bits than the 8-byte loads' % tag
        c.res['scalar = vector bits'] = 0.0
    return c.res


# ------------------------------------------------------------------ tfb_gemm_small_m
def small_m_ks(K):
    """The K-slice count of the transB kernel (<= 6 k steps per lane)."""
    return 8 if K > 768 else 4 if K > 384 else 2 if K > 192 else 1


def small_m(c, tb, M, N, K, act, bias, kind, pad=0, seed=0):
    """C[m][n] = act(sum_k A[m][k] op(B)[k][n] + bias[n]); act 0 none, 1 ReLU, 2 sigmoid. pad: extra columns of every leading
    dimension (NaN in A and B, and never written in C)."""
    dev = c.dev
    lda, ldb, ldc = K + pad, (K if tb else N) + pad, N + pad
    rb, cb = (N, K) if tb else (K, N)
    if kind == 'exact':
        r = R.exact_range(K)
        R.assert_exact(K, r / 8, r / 16, 2.0 ** -7, 0.5 if bias else 0.0, 'small_m')
        A, B = R.dyadic((M, K), r, 3, seed, dev), R.dyadic((rb, cb), r, 4, seed + 1, dev)
        b = R.dyadic((N,), 64, 7, seed + 2, dev) if bias else None
    else:
        sh = 1.5 if kind == 'shift' else 0.0
        A, B = R.gauss((M, K), seed, dev, 1.0, sh), R.gauss((rb, cb), seed + 1, dev, 1.0 / math.sqrt(K))
        b = R.gauss((N,), seed + 2, dev, 0.5) if bias else None
    Ab = torch.full((M, lda), float('nan'), device=dev)
    Ab[:, :K] = A
    Bb = torch.full((rb, ldb), float('nan'), device=dev)
    Bb[:, :cb] = B
    out = c.out((M, ldc))
    c.twice(lambda: c.call('tfb_gemm_small_m', int(tb), M, N, K, Ab, lda, Bb, ldb, out.t, ldc, b, act), [out])
    got = out.t[:, :N]
    assert bool(out.t[:, N:].isnan().all()), 'small_m wrote past column N'
    pre, mag = R.small_m(A, B, tb, b)
    tag = 'small_m %s act %d' % ('NT'[tb], act)
    if act == 2:
        err = 0.0 if kind == 'exact' else (K + 1) * R.EPS32 * mag
        s = R.sigmoid(pre)
        ratio = ((got.double() - s).abs() / R.sigmoid_allow(pre, err)).max().item()
        assert bool(torch.isfinite(got).all()) and ratio <= 1.0, '%s (%s): sigmoid %.3g x its allowance' % (tag, kind, ratio)
        c.res['%s %s' % (tag, kind)] = max(c.res.get('%s %s' % (tag, kind), 0.0), ratio)
        return c.res
    ref = pre.clamp_min(0) if act == 1 else pre
    if kind == 'exact':
        c.exact(tag, got, ref)
    else:
        c.check('%s %s' % (tag, kind), got, ref, mag, K + 1)
    return c.res


# ------------------------------------------------------------------ refusals (host-side, nothing is launched)
def refusals(c):
    """The argument checks already in the code refuse before any launch, with `argument check failed`: the batch-count and grid.y
    caps of tfb_gemm_f32_simt, M outside [1, 16] for tfb_gemm_small_m, Cin or Cout not divisible by groups and ksize not in {1, 3}
    for the convolutions. The same calls with valid arguments are accepted."""
    t = torch.zeros(64, device=c.dev)
    g = lambda M=1, N=1, K=1, bo=1, bi=1: ('tfb_gemm_f32_simt', 0, 0, M, N, K, t, max(K, 1), t, N, t, N, None, 0, 1.0, 0.0, bo, bi,
                                            0, 0, 0, 0, 0, 0)
    s = lambda M=1: ('tfb_gemm_small_m', 1, M, 1, 1, t, 1, t, 1, t, 1, None, 0)
    x, w, y = torch.zeros(4 * 4 * 6, device=c.dev), torch.zeros(6 * 6 * 25, device=c.dev), torch.zeros(4 * 4 * 6, device=c.dev)
    cf = lambda Cin=6, Cout=6, k=3, groups=3: ('tfb_conv2d_fwd', x, w, None, y, 1, 4, 4, Cin, Cout, k, 1, groups, 0)
    cd = lambda Cin=6, Cout=6, k=3, groups=3: ('tfb_conv2d_dgrad', y, w, x, 1, 4, 4, Cin, Cout, k, 1, groups)
    cw = lambda Cin=6, Cout=6, k=3, groups=3: ('tfb_conv2d_wgrad', x, y, w, None, 1, 4, 4, Cin, Cout, k, 1, groups)
    bad = {g: [dict(bo=256, bi=257), dict(bo=65536), dict(N=65535 * 64 + 1)],
           s: [dict(M=17), dict(M=0)],
           cf: [dict(Cin=5, groups=3), dict(Cout=4, groups=3), dict(k=5, groups=1), dict(k=2, groups=1)],
           cd: [dict(Cin=5, groups=3), dict(Cout=4, groups=3), dict(k=5, groups=1), dict(k=2, groups=1)],
           cw: [dict(Cin=5, groups=3), dict(Cout=4, groups=3), dict(k=5, groups=1), dict(k=7, groups=1)]}
    for make, kws in bad.items():
        for kw in kws:
            with pytest.raises(RuntimeError, match='argument check failed'):
                c.call(*make(**kw))
        c.call(*make())
    c.sync()


def pool_refusals(call, dev):
    """tfb_maxpool3x3s2_fwd / _bwd (csrc/resnet_stem.cu, the ResNet stem's max-pool) read and write four channels per access (float4
    maps, the argmax bytes as one uint32, the bf16 copy as one 8-byte store): a storage-offset view (4 bytes off 16 for the maps,
    1 to 3 bytes off 4 for the argmax, 2 bytes off 8 for the bf16 copy) is refused with `argument check failed` before anything is
    launched. The same calls on aligned operands are accepted."""
    N, H, W, C = 1, 5, 6, 4
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    n, no = N * H * W * C, N * Ho * Wo * C
    f = lambda m: torch.zeros(m + 8, device=dev)
    xb, yb, dyb, dxb = f(n), f(no), f(no), f(n)
    ab, hb = torch.zeros(no + 8, dtype=torch.uint8, device=dev), torch.zeros(no + 8, dtype=torch.bfloat16, device=dev)
    fwd = lambda x=xb[:n], y=yb[:no], y16=hb[:no], arg=ab[:no]: ('tfb_maxpool3x3s2_fwd', x, y, y16, arg, N, H, W, C)
    bwd = lambda dy=dyb[:no], arg=ab[:no], dx=dxb[:n]: ('tfb_maxpool3x3s2_bwd', dy, arg, dx, N, H, W, C)
    bad = {fwd: [dict(x=xb[1:1 + n]), dict(y=yb[1:1 + no]), dict(y16=hb[1:1 + no]), dict(arg=ab[1:1 + no]), dict(arg=ab[2:2 + no])],
           bwd: [dict(dy=dyb[1:1 + no]), dict(arg=ab[3:3 + no]), dict(dx=dxb[2:2 + n])]}
    for make, kws in bad.items():
        for kw in kws:
            with pytest.raises(RuntimeError, match='argument check failed'):
                call(*make(**kw))
        call(*make())
    call(*fwd(y16=None))                                       # the bf16 copy is optional
    if torch.device(dev).type == 'cuda':
        torch.cuda.synchronize()


# ------------------------------------------------------------------ benchmark call sites
SPIED = ('tfb_conv2d_fwd', 'tfb_conv2d_dgrad', 'tfb_conv2d_wgrad', 'tfb_gemm_f32_simt', 'tfb_gemm_small_m')
# (backbone, batch): the benchmark's configurations (bench.CONFIGS) and latentTF at the default batch
SPY_STEPS = (('transFuser', 10), ('late_fusion', 16), ('geometric_fusion', 12), ('latentTF', 10))


def _ptr(a):
    return a.data_ptr() if isinstance(a, torch.Tensor) else int(a)


def call_key(name, a):
    """What decides the kernel, the grid and the loads of one call of these entry points: the shape, the optional operands, the
    strides and the 16-byte phase (in floats) of the GEMM operands."""
    if name == 'tfb_conv2d_fwd':
        return ('fwd',) + tuple(a[4:12]) + (a[2] is not None, bool(a[12]))
    if name == 'tfb_conv2d_dgrad':
        return ('dgrad',) + tuple(a[3:11]) + (False, False)
    if name == 'tfb_conv2d_wgrad':
        return ('wgrad',) + tuple(a[4:12]) + (a[3] is not None, False)
    if name == 'tfb_gemm_f32_simt':
        return ('gemm',) + tuple(a[0:5]) + (a[6], a[8], a[10], a[11] is not None, a[12], a[13], a[14]) + tuple(a[15:23]) + \
            (_ptr(a[5]) % 16 // 4, _ptr(a[7]) % 16 // 4)
    assert name == 'tfb_gemm_small_m', name
    return ('small_m',) + tuple(a[0:4]) + (a[5], a[7], a[9], a[10] is not None, a[11])


def run_key(c, key, kind):
    """Runs the case of one call key."""
    if key[0] in CONV_OPS:
        N, H, W, Cin, Cout, k, s, g, bias, relu = key[1:]
        return conv(c, N, H, W, Cin, Cout, k, s, g, bias, relu, kind, ops=(key[0],), seed=N + H + Cin)
    if key[0] == 'gemm':
        ta, tb, M, N, Kd, lda, ldb, ldc, bias, relu, alpha, beta, bo, bi, sAo, sAi, sBo, sBi, sCo, sCi, oa, ob = key[1:]
        return gemm(c, ta, tb, M, N, Kd, kind, alpha, beta, bias, relu, lda, ldb, ldc, (bo, bi), (sAo, sAi, sBo, sBi, sCo, sCi), (oa, ob),
                    seed=M + N)
    tb, M, N, Kd, lda, ldb, ldc, bias, act = key[1:]
    assert (lda, ldb, ldc) == (Kd, Kd if tb else N, N), key
    return small_m(c, tb, M, N, Kd, act, bias, kind, seed=M + N)


def kinds_for(key):
    """Exact operands need power-of-two alpha and beta."""
    if key[0] == 'gemm' and not (_dyadic_scalar(key[11]) and _dyadic_scalar(key[12])):
        return KINDS[1:]
    return KINDS


# The calls of these entry points in one eager bf16 training step of each SPY_STEPS configuration, collected by spying on the
# C-ABI (tests/test_simt_exact.py::test_bench_call_sites_are_listed fails when a call is not in this list).
BENCH = [
    ('fwd', 10, 160, 704, 3, 32, 3, 2, 1, False, False),   # latentTF, transFuser
    ('fwd', 10, 256, 256, 3, 32, 3, 2, 1, False, False),   # latentTF, transFuser
    ('fwd', 12, 160, 704, 3, 32, 3, 2, 1, False, False),   # geometric_fusion
    ('fwd', 12, 256, 256, 3, 32, 3, 2, 1, False, False),   # geometric_fusion
    ('fwd', 16, 160, 704, 3, 32, 3, 2, 1, False, False),   # late_fusion
    ('fwd', 16, 256, 256, 3, 32, 3, 2, 1, False, False),   # late_fusion
    ('gemm', 0, 0, 40960, 64, 1, 1, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # latentTF, transFuser
    ('gemm', 0, 0, 40960, 64, 12, 12, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # latentTF, transFuser
    ('gemm', 0, 0, 40960, 64, 2, 2, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # latentTF, transFuser
    ('gemm', 0, 0, 40960, 64, 3, 3, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # latentTF, transFuser
    ('gemm', 0, 0, 49152, 64, 1, 1, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # geometric_fusion
    ('gemm', 0, 0, 49152, 64, 12, 12, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # geometric_fusion
    ('gemm', 0, 0, 49152, 64, 2, 2, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # geometric_fusion
    ('gemm', 0, 0, 49152, 64, 3, 3, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # geometric_fusion
    ('gemm', 0, 0, 65536, 64, 1, 1, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # late_fusion
    ('gemm', 0, 0, 65536, 64, 12, 12, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # late_fusion
    ('gemm', 0, 0, 65536, 64, 2, 2, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # late_fusion
    ('gemm', 0, 0, 65536, 64, 3, 3, 64, 64, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # late_fusion
    ('gemm', 0, 1, 40960, 1, 64, 64, 64, 1, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # latentTF, transFuser
    ('gemm', 0, 1, 40960, 12, 64, 64, 64, 12, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # latentTF, transFuser
    ('gemm', 0, 1, 40960, 2, 64, 64, 64, 2, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # latentTF, transFuser
    ('gemm', 0, 1, 40960, 3, 64, 64, 64, 3, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # latentTF, transFuser
    ('gemm', 0, 1, 49152, 1, 64, 64, 64, 1, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # geometric_fusion
    ('gemm', 0, 1, 49152, 12, 64, 64, 64, 12, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # geometric_fusion
    ('gemm', 0, 1, 49152, 2, 64, 64, 64, 2, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # geometric_fusion
    ('gemm', 0, 1, 49152, 3, 64, 64, 64, 3, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # geometric_fusion
    ('gemm', 0, 1, 65536, 1, 64, 64, 64, 1, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # late_fusion
    ('gemm', 0, 1, 65536, 12, 64, 64, 64, 12, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # late_fusion
    ('gemm', 0, 1, 65536, 2, 64, 64, 64, 2, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # late_fusion
    ('gemm', 0, 1, 65536, 3, 64, 64, 64, 3, True, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # late_fusion
    ('gemm', 1, 0, 128, 256, 10, 128, 256, 256, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # latentTF, transFuser
    ('gemm', 1, 0, 128, 256, 12, 128, 256, 256, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # geometric_fusion
    ('gemm', 1, 0, 128, 256, 16, 128, 256, 256, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # late_fusion
    ('gemm', 1, 0, 256, 512, 10, 256, 512, 512, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # latentTF, transFuser
    ('gemm', 1, 0, 256, 512, 12, 256, 512, 512, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # geometric_fusion
    ('gemm', 1, 0, 256, 512, 16, 256, 512, 512, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # late_fusion
    ('gemm', 1, 0, 64, 128, 10, 64, 128, 128, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # latentTF, transFuser
    ('gemm', 1, 0, 64, 128, 12, 64, 128, 128, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # geometric_fusion
    ('gemm', 1, 0, 64, 128, 16, 64, 128, 128, False, 0, 1.0, 0.0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0),   # late_fusion
    ('small_m', 0, 10, 128, 64, 64, 128, 128, False, 0),   # latentTF, transFuser
    ('small_m', 0, 10, 256, 128, 128, 256, 256, False, 0),   # latentTF, transFuser
    ('small_m', 0, 10, 512, 256, 256, 512, 512, False, 0),   # latentTF, transFuser
    ('small_m', 0, 12, 128, 64, 64, 128, 128, False, 0),   # geometric_fusion
    ('small_m', 0, 12, 256, 128, 128, 256, 256, False, 0),   # geometric_fusion
    ('small_m', 0, 12, 512, 256, 256, 512, 512, False, 0),   # geometric_fusion
    ('small_m', 0, 16, 128, 64, 64, 128, 128, False, 0),   # late_fusion
    ('small_m', 0, 16, 256, 128, 128, 256, 256, False, 0),   # late_fusion
    ('small_m', 0, 16, 512, 256, 256, 512, 512, False, 0),   # late_fusion
    ('small_m', 1, 10, 128, 256, 256, 256, 128, True, 1),   # latentTF, transFuser
    ('small_m', 1, 10, 144, 1512, 1512, 1512, 144, True, 1),   # latentTF, transFuser
    ('small_m', 1, 10, 144, 576, 576, 576, 144, True, 1),   # latentTF, transFuser
    ('small_m', 1, 10, 1512, 144, 144, 144, 1512, True, 2),   # latentTF, transFuser
    ('small_m', 1, 10, 18, 216, 216, 216, 18, True, 1),   # latentTF, transFuser
    ('small_m', 1, 10, 18, 72, 72, 72, 18, True, 1),   # latentTF, transFuser
    ('small_m', 1, 10, 216, 18, 18, 18, 216, True, 2),   # latentTF, transFuser
    ('small_m', 1, 10, 216, 54, 54, 54, 216, True, 2),   # latentTF, transFuser
    ('small_m', 1, 10, 256, 512, 512, 512, 256, True, 1),   # latentTF, transFuser
    ('small_m', 1, 10, 54, 216, 216, 216, 54, True, 1),   # latentTF, transFuser
    ('small_m', 1, 10, 54, 576, 576, 576, 54, True, 1),   # latentTF, transFuser
    ('small_m', 1, 10, 576, 144, 144, 144, 576, True, 2),   # latentTF, transFuser
    ('small_m', 1, 10, 576, 54, 54, 54, 576, True, 2),   # latentTF, transFuser
    ('small_m', 1, 10, 64, 128, 128, 128, 64, True, 1),   # latentTF, transFuser
    ('small_m', 1, 10, 72, 18, 18, 18, 72, True, 2),   # latentTF, transFuser
    ('small_m', 1, 10, 72, 8, 8, 8, 72, True, 2),   # latentTF, transFuser
    ('small_m', 1, 10, 8, 72, 72, 72, 8, True, 1),   # latentTF, transFuser
    ('small_m', 1, 12, 128, 256, 256, 256, 128, True, 1),   # geometric_fusion
    ('small_m', 1, 12, 144, 1512, 1512, 1512, 144, True, 1),   # geometric_fusion
    ('small_m', 1, 12, 144, 576, 576, 576, 144, True, 1),   # geometric_fusion
    ('small_m', 1, 12, 1512, 144, 144, 144, 1512, True, 2),   # geometric_fusion
    ('small_m', 1, 12, 18, 216, 216, 216, 18, True, 1),   # geometric_fusion
    ('small_m', 1, 12, 18, 72, 72, 72, 18, True, 1),   # geometric_fusion
    ('small_m', 1, 12, 216, 18, 18, 18, 216, True, 2),   # geometric_fusion
    ('small_m', 1, 12, 216, 54, 54, 54, 216, True, 2),   # geometric_fusion
    ('small_m', 1, 12, 256, 512, 512, 512, 256, True, 1),   # geometric_fusion
    ('small_m', 1, 12, 54, 216, 216, 216, 54, True, 1),   # geometric_fusion
    ('small_m', 1, 12, 54, 576, 576, 576, 54, True, 1),   # geometric_fusion
    ('small_m', 1, 12, 576, 144, 144, 144, 576, True, 2),   # geometric_fusion
    ('small_m', 1, 12, 576, 54, 54, 54, 576, True, 2),   # geometric_fusion
    ('small_m', 1, 12, 64, 128, 128, 128, 64, True, 1),   # geometric_fusion
    ('small_m', 1, 12, 72, 18, 18, 18, 72, True, 2),   # geometric_fusion
    ('small_m', 1, 12, 72, 8, 8, 8, 72, True, 2),   # geometric_fusion
    ('small_m', 1, 12, 8, 72, 72, 72, 8, True, 1),   # geometric_fusion
    ('small_m', 1, 16, 128, 256, 256, 256, 128, True, 1),   # late_fusion
    ('small_m', 1, 16, 144, 1512, 1512, 1512, 144, True, 1),   # late_fusion
    ('small_m', 1, 16, 144, 576, 576, 576, 144, True, 1),   # late_fusion
    ('small_m', 1, 16, 1512, 144, 144, 144, 1512, True, 2),   # late_fusion
    ('small_m', 1, 16, 18, 216, 216, 216, 18, True, 1),   # late_fusion
    ('small_m', 1, 16, 18, 72, 72, 72, 18, True, 1),   # late_fusion
    ('small_m', 1, 16, 216, 18, 18, 18, 216, True, 2),   # late_fusion
    ('small_m', 1, 16, 216, 54, 54, 54, 216, True, 2),   # late_fusion
    ('small_m', 1, 16, 256, 512, 512, 512, 256, True, 1),   # late_fusion
    ('small_m', 1, 16, 54, 216, 216, 216, 54, True, 1),   # late_fusion
    ('small_m', 1, 16, 54, 576, 576, 576, 54, True, 1),   # late_fusion
    ('small_m', 1, 16, 576, 144, 144, 144, 576, True, 2),   # late_fusion
    ('small_m', 1, 16, 576, 54, 54, 54, 576, True, 2),   # late_fusion
    ('small_m', 1, 16, 64, 128, 128, 128, 64, True, 1),   # late_fusion
    ('small_m', 1, 16, 72, 18, 18, 18, 72, True, 2),   # late_fusion
    ('small_m', 1, 16, 72, 8, 8, 8, 72, True, 2),   # late_fusion
    ('small_m', 1, 16, 8, 72, 72, 72, 8, True, 1),   # late_fusion
    ('wgrad', 1, 40960, 1, 64, 1, 1, 1, 1, False, False),   # latentTF, transFuser
    ('wgrad', 1, 40960, 1, 64, 12, 1, 1, 1, False, False),   # latentTF, transFuser
    ('wgrad', 1, 40960, 1, 64, 2, 1, 1, 1, False, False),   # latentTF, transFuser
    ('wgrad', 1, 40960, 1, 64, 3, 1, 1, 1, False, False),   # latentTF, transFuser
    ('wgrad', 1, 49152, 1, 64, 1, 1, 1, 1, False, False),   # geometric_fusion
    ('wgrad', 1, 49152, 1, 64, 12, 1, 1, 1, False, False),   # geometric_fusion
    ('wgrad', 1, 49152, 1, 64, 2, 1, 1, 1, False, False),   # geometric_fusion
    ('wgrad', 1, 49152, 1, 64, 3, 1, 1, 1, False, False),   # geometric_fusion
    ('wgrad', 1, 65536, 1, 64, 1, 1, 1, 1, False, False),   # late_fusion
    ('wgrad', 1, 65536, 1, 64, 12, 1, 1, 1, False, False),   # late_fusion
    ('wgrad', 1, 65536, 1, 64, 2, 1, 1, 1, False, False),   # late_fusion
    ('wgrad', 1, 65536, 1, 64, 3, 1, 1, 1, False, False),   # late_fusion
    ('wgrad', 10, 160, 704, 3, 32, 3, 2, 1, False, False),   # latentTF, transFuser
    ('wgrad', 10, 256, 256, 3, 32, 3, 2, 1, False, False),   # latentTF, transFuser
    ('wgrad', 12, 160, 704, 3, 32, 3, 2, 1, False, False),   # geometric_fusion
    ('wgrad', 12, 256, 256, 3, 32, 3, 2, 1, False, False),   # geometric_fusion
    ('wgrad', 16, 160, 704, 3, 32, 3, 2, 1, False, False),   # late_fusion
    ('wgrad', 16, 256, 256, 3, 32, 3, 2, 1, False, False),   # late_fusion
]
