"""The exact-fp32 CUDA-core convolution and GEMM kernels (csrc/conv_simt.cu, csrc/gemm_simt.cu) under the CPU emulation (2 SMs), at
reduced sizes that still cross every dispatch boundary: the forward's CO_T = 8 / 16 / 24 / 32 and the dgrad's CI_T choice, channel
counts across the 32-channel chunk, k = 1 and 3, stride 2 with both parities of H and W, H = W = 1, groups 1 / 3 / 9; the three
weight-gradient kernels with one pixel split and several, the fused fold and the grid-wide one; every GEMM layout with the 8-byte
and the scalar loads at the 128 x 64 x 16 tile edges, K = 0, strided windows and two-level batches; the small-M K-slice
thresholds. Also the max-pool's refusal of misaligned operands (csrc/resnet_stem.cu). Cases: tests/simt_cases.py; on the H100 at full size: tests/test_simt_exact.py."""
import pytest

import simt_cases as K
from cuda_emul import loader

SMS = 2
# (N, H, W, Cin, Cout, k, stride, groups, bias, relu)
EMUL_CONV = [
    (1, 5, 7, 33, 9, 3, 1, 1, True, True),          # Cig 33: a partial chunk; CO_T 16
    (1, 5, 7, 32, 7, 3, 2, 1, False, False),        # stride 2, odd H / W; CO_T 8
    (1, 6, 8, 31, 17, 3, 2, 1, True, False),        # stride 2, even H / W; Cog 17: CO_T 32
    (1, 5, 5, 65, 24, 3, 1, 1, False, True),        # Cig 65; CO_T 24
    (1, 4, 6, 64, 65, 3, 1, 1, True, False),        # Cog 65 (the dgrad's partial chunk)
    (1, 1, 1, 16, 40, 3, 1, 1, True, True),         # H = W = 1: the centre tap only
    (1, 1, 1, 8, 1, 3, 2, 1, False, False),
    (1, 5, 7, 72, 72, 3, 1, 3, True, True),         # groups 3 (24 per group): CO_T / CI_T 24, dbias with groups
    (1, 5, 6, 216, 216, 3, 2, 9, True, False),      # groups 9, stride 2
    (1, 4, 5, 27, 48, 3, 1, 3, False, False),       # 9 -> 16 per group
    (1, 7, 9, 40, 48, 1, 2, 1, False, False),       # strided 1x1 shortcut, odd H / W
    (2, 6, 5, 17, 72, 1, 2, 1, True, False),        # strided 1x1, even H, odd W
    (1, 13, 22, 64, 64, 3, 1, 1, True, False),      # generic wgrad: 36864 weights (grid-wide fold), 2 splits, 286 pixels
    (1, 15, 20, 72, 72, 3, 1, 3, True, False),      # generic wgrad: 15552 weights (fused fold), 2 splits
    (1, 5, 7, 3, 8, 3, 1, 1, True, True),           # small-Cin wgrad ...
    (1, 9, 8, 1, 32, 3, 2, 1, False, False),
    (2, 12, 13, 4, 40, 3, 1, 1, True, False),       # ... 2 splits
    (2, 25, 31, 2, 64, 3, 2, 1, False, False),      # ... stride 2, 2 splits
    (1, 127, 1, 64, 1, 1, 1, 1, True, False),       # narrow-out wgrad: 127 pixels, one split
    (1, 129, 1, 70, 2, 1, 1, 1, False, False),      # ... 2 splits, the last of one pixel
    (1, 11, 47, 100, 3, 1, 1, 1, True, False),      # ... 144-pixel splits (16-pixel rounding), a partial last one
    (2, 16, 40, 64, 12, 1, 1, 1, False, False),     # ... 8 splits
    (1, 9, 15, 130, 16, 1, 1, 1, True, True),       # ... 3 channel blocks
]
EMUL_CONV_KINDS = [(s, kind) for i, s in enumerate(EMUL_CONV) for kind in (K.KINDS if i % 3 == 0 else ('exact', K.KINDS[1 + i % 2]))]

# (M, N, K, kind, alpha, beta, bias, relu, extra) with extra: lda / ldb / ldc padding, batch, strides, offs
EMUL_GEMM = [
    (129, 65, 17, 'exact', 0.5, 0.25, True, True, {}),
    (127, 63, 16, 'gauss', 1.0, 0.0, False, False, {}),
    (128, 64, 15, 'shift', -2.0, 1.0, True, False, {}),
    (5, 3, 1, 'exact', 1.0, 1.0, False, False, {}),
    (33, 20, 0, 'exact', 1.0, 1.0, True, False, {}),           # K = 0: beta * C + bias
    (33, 20, 0, 'exact', 1.0, 0.0, False, True, {}),           # K = 0 into a NaN-filled C
    (40, 24, 16, 'exact', 1.0, 0.0, False, False, dict(pad=(6, 10, 3), offs=(2, 6))),    # column windows, 8-byte aligned
    (37, 70, 33, 'gauss', 1.0, 0.0, True, False, dict(pad=(1, 3, 0))),                   # odd leading dimensions: scalar loads
    (17, 9, 24, 'exact', 0.5, 1.0, False, False, dict(batch=(2, 3), gap=2, offs=(2, 2))),   # two-level batch, 8-byte head offsets
    (20, 16, 31, 'gauss', 1.0, 0.0, False, False, dict(batch=(3, 2), gap=1, offs=(1, 0))),
]
LAYOUTS = [(0, 0), (0, 1), (1, 0), (1, 1)]

# (transB, M, N, K, act, bias)
EMUL_SMALL_M = [(1, 1, 9, 192, 0, True), (1, 10, 9, 193, 1, False), (1, 16, 5, 384, 2, True), (1, 3, 7, 385, 0, False),
                (1, 16, 3, 768, 1, True), (1, 10, 11, 769, 2, False), (1, 1, 2, 40, 2, True), (1, 16, 33, 5, 0, True),
                (0, 1, 33, 1, 0, True), (0, 10, 70, 5, 1, False), (0, 16, 40, 7, 2, True), (0, 3, 31, 9, 0, False),
                (0, 16, 64, 200, 1, True)]


@pytest.fixture(scope='module')
def ctx():
    return K.Ctx(loader.emul().call, 'cpu', SMS)


def _show(what, res):
    print('%s: %s' % (what, {k: '%.4f' % v for k, v in res.items()}))


def _fresh(ctx):
    ctx.res = {}
    return ctx


def gemm_args(M, N, Kd, ta, tb, extra):
    """Keyword arguments of simt_cases.gemm from a compact description: pad (lda, ldb, ldc extra columns), batch with `gap` floats
    between consecutive matrices, offs."""
    pa, pb, pc = extra.get('pad', (0, 0, 0))
    lda, ldb, ldc = (M if ta else Kd) + pa, (Kd if tb else N) + pb, N + pc
    kw = dict(lda=lda, ldb=ldb, ldc=ldc, offs=extra.get('offs', (0, 0)))
    if 'batch' in extra:
        bo, bi = extra['batch']
        gap = extra['gap']
        sAi, sBi, sCi = (Kd if ta else M) * lda + gap, (N if tb else Kd) * ldb + gap, M * ldc + gap
        kw.update(batch=(bo, bi), strides=(bi * sAi + gap, sAi, bi * sBi + gap, sBi, bi * sCi + gap, sCi))
    return kw


@pytest.mark.parametrize('shape,kind', EMUL_CONV_KINDS)
def test_conv_emulated(ctx, shape, kind):
    _show('conv %s %s' % (shape, kind), K.conv(_fresh(ctx), *shape, kind, seed=sum(shape[:8])))


def test_conv_cases_reach_every_wgrad_path():
    """The emulated shapes reach each weight-gradient kernel with one pixel split and with several, and both folds of the
    generic kernel."""
    seen = set()
    for s in EMUL_CONV:
        kern, splits, fused = K.wgrad_path(*s[:8], SMS)
        seen.add((kern, splits > 1))
        if kern == 'generic':
            seen.add(('generic fold', fused))
    want = {(k, m) for k in ('generic', 'smallcin', 'narrowout') for m in (False, True)} | {('generic fold', True), ('generic fold', False)}
    assert want <= seen, sorted(want - seen)


@pytest.mark.parametrize('ta,tb', LAYOUTS)
@pytest.mark.parametrize('M,N,Kd,kind,alpha,beta,bias,relu,extra', EMUL_GEMM)
def test_gemm_emulated(ctx, ta, tb, M, N, Kd, kind, alpha, beta, bias, relu, extra):
    _show('gemm ta %d tb %d M %d N %d K %d %s' % (ta, tb, M, N, Kd, kind),
          K.gemm(_fresh(ctx), ta, tb, M, N, Kd, kind, alpha, beta, bias, relu, seed=M + N + Kd, **gemm_args(M, N, Kd, ta, tb, extra)))


@pytest.mark.parametrize('kind', K.KINDS)
@pytest.mark.parametrize('tb,M,N,Kd,act,bias', EMUL_SMALL_M)
def test_small_m_emulated(ctx, tb, M, N, Kd, act, bias, kind):
    _show('small_m tb %d M %d N %d K %d act %d %s' % (tb, M, N, Kd, act, kind),
          K.small_m(_fresh(ctx), tb, M, N, Kd, act, bias, kind, pad=3 if M == 10 else 0, seed=M + N + Kd))


def test_small_m_cases_reach_every_k_slice():
    assert {K.small_m_ks(k) for tb, _, _, k, _, _ in EMUL_SMALL_M if tb} == {1, 2, 4, 8}


def test_argument_checks_emulated(ctx):
    K.refusals(ctx)


def test_pool_misaligned_operands_refused_emulated():
    from cuda_emul import stem_emul
    K.pool_refusals(stem_emul.call, 'cpu')
