"""The normalisation kernels of csrc/norm.cu under the CPU emulation (2 SMs), at reduced sizes that still cross every dispatch
boundary: the flat column reduction (C / 4 <= 128, M >= 4096) and the 128-channel slabs, odd tails of the two-rows-in-flight loop,
the flat and grid pooled apply passes (HW >= 1024), C parities of the final fold, the scalar column sum. Cases: tests/norm_cases.py;
on the H100 at full size: tests/test_norm_exact.py."""
import pytest

import norm_cases as K
from cuda_emul import loader

SMS = 2
EMUL_BN = [(4, 4096, 30.0, 'relu'), (8, 4097, 0.0, 'residual'), (72, 4095, 10.0, 'y16'), (72, 4096, 30.0, 'plain'),
           (216, 4097, 10.0, 'relu'), (512, 33, 30.0, 'y16'),
           (516, 7, 0.0, 'relu'), (576, 9, 30.0, 'residual'), (1512, 1, 10.0, 'plain'), (2048, 9, 0.0, 'y16'), (516, 300, 10.0, 'relu')]
EMUL_STATS = [(72, 1024, 3, 'pool'), (72, 1023, 1, 'pool'), (72, 1, 10, 'pool'), (516, 3, 3, 'pool'), (2048, 2, 3, 'pool'),
              (72, 110, 3, 'residual'), (516, 7, 3, 'y16'), (1512, 3, 1, 'plain'), (2048, 1, 3, 'residual')]
EMUL_POOL = [(72, 1024, 1), (8, 110, 3), (516, 3, 10), (2048, 1, 3)]
EMUL_SE = [(72, 1, 4100), (72, 3, 1367), (216, 110, 38), (72, 1024, 4), (576, 3, 3), (1512, 110, 2)]
EMUL_COLSUM = [(1, 4096, 'dense'), (3, 300, 'padded'), (7, 4097, 'dense'), (12, 4096, 'dense'), (12, 200, 'padded'), (64, 4096, 'offset'),
               (648, 40, 'padded'), (648, 33, 'dense'), (64, 4100, 'padded')]
EMUL_GRAD_PREP = [(1, 1, ('g32', 'g16', 'dbias'), True), (7, 1740, ('g32',), True), (216, 1740, ('g16',), False),
                  (648, 60, ('dbias',), True), (4536, 9, ('g32', 'g16', 'dbias'), True), (7, 30000, ('dbias',), False)]
EMUL_LN = [(72, 24, False), (216, 1, True), (576, 17, False), (1512, 9, True), (1, 20, False), (31, 130, True), (257, 9, False),
           (2049, 3, False)]
EMUL_ADLN = [(72, 24, 0.1, True), (216, 17, 0.0, False), (1512, 5, 0.1, False), (31, 9, 0.1, True), (2049, 2, 0.0, True)]


@pytest.fixture(scope='module')
def ctx():
    return K.Ctx(loader.emul().call, 'cpu', SMS)


def _show(what, res):
    print('%s: %s' % (what, {k: '%.4f' % v if 'rel err' not in k else '%.2e' % v for k, v in res.items()}))


def _fresh(ctx):
    ctx.res = {}
    return ctx


@pytest.mark.parametrize('C,M,shift,variant', EMUL_BN)
def test_bn_train_emulated(ctx, C, M, shift, variant):
    _show('bn C %d M %d shift %g %s' % (C, M, shift, variant), K.bn_train(_fresh(ctx), C, M, shift, variant))


@pytest.mark.parametrize('C,HW,nb,variant', EMUL_STATS)
def test_bn_fwd_stats_emulated(ctx, C, HW, nb, variant):
    _show('bn_fwd_stats C %d HW %d x %d %s' % (C, HW, nb, variant), K.bn_fwd_stats(_fresh(ctx), C, HW, nb, variant))


@pytest.mark.parametrize('C,HW,nb', EMUL_POOL)
def test_bn_fwd_pool_emulated(ctx, C, HW, nb):
    _show('bn_fwd pool C %d HW %d x %d' % (C, HW, nb), K.bn_fwd_pool(_fresh(ctx), C, HW, nb))


@pytest.mark.parametrize('C,hw,nb', EMUL_SE)
def test_bn_bwd_se_emulated(ctx, C, hw, nb):
    _show('bn_bwd_se C %d hw %d x %d' % (C, hw, nb), K.bn_bwd_se(_fresh(ctx), C, hw, nb, side=hw == 3))


@pytest.mark.parametrize('variant', ['relu', 'residual', 'y16'])
@pytest.mark.parametrize('C', [8, 216, 1512])
def test_bn_apply_emulated(ctx, C, variant):
    _show('bn_apply C %d %s' % (C, variant), K.bn_apply(_fresh(ctx), C, 37, variant))


@pytest.mark.parametrize('C,M,layout', EMUL_COLSUM)
def test_colsum_emulated(ctx, C, M, layout):
    _show('colsum C %d M %d %s' % (C, M, layout), K.colsum(_fresh(ctx), C, M, layout))


@pytest.mark.parametrize('C,M,outs,relu', EMUL_GRAD_PREP)
def test_grad_prep_emulated(ctx, C, M, outs, relu):
    _show('grad_prep C %d M %d %s relu %d' % (C, M, outs, relu), K.grad_prep(_fresh(ctx), C, M, outs, relu))


@pytest.mark.parametrize('C,R,acc', EMUL_LN)
def test_layernorm_emulated(ctx, C, R, acc):
    _show('layernorm C %d R %d acc %d' % (C, R, acc), K.layernorm(_fresh(ctx), C, R, acc))


@pytest.mark.parametrize('C,R,p,gx', EMUL_ADLN)
def test_add_dropout_ln_emulated(ctx, C, R, p, gx):
    _show('add_dropout_ln C %d R %d p %g gx %d' % (C, R, p, gx), K.add_dropout_ln(_fresh(ctx), C, R, p, gx))


def test_stream_reuse_emulated(ctx):
    K.stream_reuse(ctx, [(K.bn_train, (72, 4096, 10.0, 'relu')), (K.colsum, (7, 300, 'padded')), (K.layernorm, (257, 9, False)),
                         (K.bn_bwd_se, (576, 3, 3)), (K.grad_prep, (648, 60, ('dbias',), True)), (K.bn_train, (516, 7, 0.0, 'residual')),
                         (K.bn_fwd_pool, (8, 110, 3)), (K.add_dropout_ln, (31, 9, 0.1, True))])


def test_misaligned_operands_refused_emulated(ctx):
    K.refusals(ctx)
