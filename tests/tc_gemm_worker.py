"""Worker of tests/test_tc_exact.py::test_gemm_bf16_exact: runs the bf16 tensor-core GEMM entry points at one forced tile width and
prints one JSON line {"width": ..., "cases": [{"case", "rel", "ratio", "error"}]}.

The tile width is fixed per process (TFB_GEMM_BN is read once, on the first launch), so the parent starts one worker per width.
Every output is pre-filled with NaN inside a larger buffer filled with a sentinel; every case runs twice and must give the same bits.
Usage: python tests/tc_gemm_worker.py WIDTH   (with TFB_GEMM_BN=WIDTH in the environment)."""
import json
import os
import sys
import traceback

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402

import tc_ref as R  # noqa: E402
from transfuser_b200 import _lib  # noqa: E402

DEV = 'cuda'
SENT = -1024.0           # sentinel outside the output views (exactly representable in bf16 and fp32)
TOL = 3e-5               # relative L2 against the exact-operand reference: 10x the measured worst, 3.2e-6 (K = 6048)
N_RAGGED = 234           # ragged against every tile width: 234 = 7*32 + 10 = 3*64 + 42 = 2*96 + 42 = 128 + 106 = 160 + 74 = 192 + 42


def call(name, *a):
    _lib.call(name, *a)


def operand(rows, cols, gen, ld_extra=0):
    """bf16 [rows, cols] view with a leading dimension rounded up to 8 elements (16-byte TMA rows) plus ld_extra."""
    ld = (cols + 7) // 8 * 8 + ld_extra
    buf = torch.randn(rows, ld, device=DEV, generator=gen).bfloat16()
    return buf[:, :cols], ld


class Out:
    """Output view [M, N] (leading dimension ld, column offset col0) inside a sentinel-filled buffer."""

    def __init__(self, M, N, ld=None, col0=0, dtype=torch.float32, nbatch=1):
        self.ld = ld or (N + 3) // 4 * 4 + 4                # default: 16-byte rows (the coalesced epilogue path)
        assert self.ld >= col0 + N
        self.buf = torch.full((nbatch, M + 1, self.ld), SENT, dtype=dtype, device=DEV)
        self.v = self.buf[:, :M, col0:col0 + N]
        self.M, self.N, self.col0, self.nbatch = M, N, col0, nbatch

    def fill(self, val=None):
        self.buf.fill_(SENT)
        if val is None:
            self.v.fill_(float('nan'))
        else:
            self.v.copy_(val)
        return self

    def ptr(self):
        return self.v.data_ptr()

    def outside_ok(self):
        mask = torch.ones_like(self.buf, dtype=torch.bool)
        mask[:, :self.M, self.col0:self.col0 + self.N] = False
        return bool((self.buf[mask] == SENT).all())

    def bits(self):
        return self.buf.clone().view(torch.int16 if self.buf.dtype == torch.bfloat16 else torch.int32)


def ref_gemm(a, b, ta, tb, alpha, bias, beta, c0, relu):
    A = a.double().t() if ta else a.double()
    B = b.double().t() if tb else b.double()
    r, mag = A @ B, A.abs() @ B.abs()
    r, mag = alpha * r, abs(alpha) * mag
    if bias is not None:
        r, mag = r + bias.double(), mag + bias.double().abs()
    if beta:
        r, mag = r + beta * c0.double(), mag + abs(beta) * c0.double().abs()
    if relu:
        r = r.clamp_min(0)
    return r, mag


def twice(launch, out):
    """Runs launch() twice on a freshly pre-filled output; the two runs must give the same bits; returns the first run's buffer."""
    res = []
    for _ in range(2):
        out.fill(getattr(out, 'init', None))
        launch()
        torch.cuda.synchronize()
        assert out.outside_ok(), 'write outside the output view'
        res.append(out.bits())
    assert torch.equal(res[0], res[1]), 'two launches differ'
    return out


def main(width):
    gen = torch.Generator(device=DEV).manual_seed(1000 + width)
    cases = []

    def case(name, fn):
        try:
            rel, ratio = fn()
            cases.append(dict(case=name, rel=rel, ratio=ratio, error=None))
        except Exception as e:           # reported to the parent test, which fails on it
            cases.append(dict(case=name, rel=None, ratio=None, error='%s: %s' % (type(e).__name__, str(e)[:600]),
                              tb=traceback.format_exc()[-1500:]))

    def plain(M, N, K, ta, tb, alpha=1.0, bias=False, relu=False, beta=0.0, splits=1, ldc=None, col0=0, cap=None):
        a, lda = operand(K if ta else M, M if ta else K, gen)
        b, ldb = operand(N if tb else K, K if tb else N, gen)
        bv = torch.randn(N, device=DEV, generator=gen) if bias else None
        out = Out(M, N, ldc, col0)
        c0 = torch.randn(M, N, device=DEV, generator=gen) if beta else None
        out.init = c0[None] if beta else None

        def launch():
            call('tfb_gemm_bf16_tc', int(ta), int(tb), M, N, K, a.data_ptr(), lda, b.data_ptr(), ldb, out.ptr(), out.ld, bv,
                 int(relu), float(alpha), float(beta), splits)
        twice(launch, out)
        r, mag = ref_gemm(a, b, ta, tb, alpha, bv, beta, c0, relu)
        res = R.check(out.v[0], r, mag, K + splits + 3, TOL, what='gemm ta%d tb%d M%d N%d K%d' % (ta, tb, M, N, K))
        return res, out, (a, lda, b, ldb, bv)

    # all four layouts, alpha != 1, bias
    for ta, tb in ((0, 1), (0, 0), (1, 0), (1, 1)):
        case('layout ta%d tb%d' % (ta, tb), lambda ta=ta, tb=tb: plain(129, N_RAGGED, 72, ta, tb, alpha=0.75, bias=True)[0])
    # M across the 128-row tile boundary, short and long contractions, fused bias + ReLU
    for M, K in ((32, 24), (127, 1512), (128, 16), (129, 24), (1740, 1512)):
        case('M%d K%d bias relu' % (M, K), lambda M=M, K=K: plain(M, N_RAGGED, K, 0, 1, bias=True, relu=True)[0])
    case('M70400 K16 dgrad form', lambda: plain(70400, N_RAGGED, 16, 0, 0)[0])
    # split-K (explicit and automatic; the bias must be added once), beta = 1 accumulation, the scalar read-modify-write path
    num_kb = (6048 + 63) // 64
    for s in (2, 3, num_kb, 0):
        case('wgrad form K6048 splits %d bias' % s, lambda s=s: plain(72, N_RAGGED, 6048, 1, 0, bias=True, splits=s)[0])
    case('K6048 splits 3 beta 1', lambda: plain(72, N_RAGGED, 6048, 1, 0, beta=1.0, splits=3)[0])
    case('beta 1 accumulate', lambda: plain(300, N_RAGGED, 72, 0, 1, beta=1.0)[0])
    case('beta 1 relu (scalar path)', lambda: plain(300, N_RAGGED, 72, 0, 1, beta=1.0, relu=True, bias=True)[0])
    case('ldc % 4 != 0 (scalar path)', lambda: plain(300, N_RAGGED, 72, 0, 1, ldc=N_RAGGED + 3, bias=True, relu=True)[0])
    case('unaligned view (scalar path)', lambda: plain(300, N_RAGGED, 72, 1, 0, ldc=240, col0=1, bias=True)[0])

    # grid cap: bitwise identical to the uncapped launch at the same width and split count
    def capped(ta, tb, K, splits):
        res, out, (a, lda, b, ldb, bv) = plain(1740 if not ta else 200, N_RAGGED, K, ta, tb, bias=True, splits=splits)
        ref_bits = out.bits()
        try:
            for cap in (1, 7, 33):
                call('tfb_gemm_set_max_ctas', cap)
                twice(lambda: call('tfb_gemm_bf16_tc', ta, tb, out.M, N_RAGGED, K, a.data_ptr(), lda, b.data_ptr(), ldb, out.ptr(), out.ld,
                                   bv, 0, 1.0, 0.0, splits), out)
                assert torch.equal(out.bits(), ref_bits), 'max_ctas %d changed the result' % cap
        finally:
            call('tfb_gemm_set_max_ctas', 0)
        return res
    case('max_ctas 1/7/33 splits 1', lambda: capped(0, 1, 1512, 1))
    case('max_ctas 1/7/33 splits 3', lambda: capped(1, 0, 6048, 3))

    # bf16 output: the same bits as bf16(fp32 launch)
    def out16(tb):
        M, K = 1740, 216
        res, o32, (a, lda, b, ldb, bv) = plain(M, N_RAGGED, K, 0, tb, alpha=1.25, bias=True, relu=True)
        o16 = Out(M, N_RAGGED, 240, dtype=torch.bfloat16)
        twice(lambda: call('tfb_gemm_bf16_tc_out16', tb, M, N_RAGGED, K, a.data_ptr(), lda, b.data_ptr(), ldb, o16.ptr(), o16.ld, bv, 1,
                           1.25), o16)
        assert torch.equal(o16.v[0].view(torch.int16), o32.v[0].bfloat16().view(torch.int16)), 'out16 != bf16(fp32 output)'
        return res
    case('out16 tb1', lambda: out16(1))
    case('out16 tb0', lambda: out16(0))

    # column statistics: two calls without zeroing give exactly twice the sums; the sums against fp64 sums of the kernel's output
    def stats():
        M, K = 1740, 216
        a, lda = operand(M, K, gen)
        b, ldb = operand(N_RAGGED, K, gen)
        out = Out(M, N_RAGGED)
        st = torch.zeros(2 * N_RAGGED, dtype=torch.float64, device=DEV)
        snaps = []
        for _ in range(2):
            out.fill()
            call('tfb_gemm_bf16_tc_stats', M, N_RAGGED, K, a.data_ptr(), lda, b.data_ptr(), ldb, out.ptr(), out.ld, st)
            torch.cuda.synchronize()
            assert out.outside_ok()
            snaps.append(st.clone())
        assert torch.equal(snaps[1], 2 * snaps[0]), 'second statistics call did not exactly double the sums'
        y = out.v[0].double()
        r, mag = ref_gemm(a, b, False, True, 1.0, None, 0.0, None, False)
        res = R.check(out.v[0], r, mag, K + 3, TOL, what='stats gemm output')
        R.check(snaps[0][:N_RAGGED], y.sum(0), y.abs().sum(0), M + 8, 1e-4, what='column sums')
        R.check(snaps[0][N_RAGGED:], (y * y).sum(0), (y * y).sum(0), M + 8, 1e-4, what='column sums of squares')
        return res
    case('stats x2', stats)

    # batched grouped-conv weight gradient: per-batch column windows of the same two matrices
    def wgrad(nbatch, splits):
        M, N, K = 24, 216, 1000
        a, lda = operand(K, nbatch * M + 8, gen)       # dy windows [K, M] at column b * a_step
        b, ldb = operand(K, nbatch * N + 8, gen)       # im2col windows [K, N] at column b * b_step
        a_step, b_step = M, N
        out = Out(M, N, nbatch=nbatch)
        twice(lambda: call('tfb_gemm_bf16_tc_wgrad_batched', M, N, K, a.data_ptr(), lda, a_step, b.data_ptr(), ldb, b_step, out.ptr(),
                           out.ld, out.buf.stride(0), nbatch, splits), out)
        worst = (0.0, 0.0)
        for i in range(nbatch):
            r, mag = ref_gemm(a[:, i * a_step:i * a_step + M], b[:, i * b_step:i * b_step + N], True, False, 1.0, None, 0.0, None, False)
            res = R.check(out.v[i], r, mag, K + 64, TOL, what='wgrad batch %d' % i)
            worst = (max(worst[0], res[0]), max(worst[1], res[1]))
        return worst
    for nb in (1, 3, 32):
        for s in (0, 4):
            case('wgrad_batched nbatch %d splits %d' % (nb, s), lambda nb=nb, s=s: wgrad(nb, s))
    return cases


if __name__ == '__main__':
    w = int(sys.argv[1])
    assert os.environ.get('TFB_GEMM_BN') == str(w), 'run with TFB_GEMM_BN set to the width'
    torch.cuda.set_device(0)
    print(json.dumps(dict(width=w, cases=main(w))))
