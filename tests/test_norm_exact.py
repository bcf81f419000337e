"""The normalisation kernels of csrc/norm.cu on the H100 at full size, against the float64 references of tests/norm_ref.py
(cases: tests/norm_cases.py; the same cases at reduced size under the CPU emulation: tests/test_norm_emulated.py). Every case
runs twice into NaN-filled, sentinel-guarded outputs and must give the same bits, and must leave sums_ws all zero. Each test
prints its worst allowance ratio per check (1.0 = at the bound), and the BatchNorm cases the worst relative invstd error per
mean / std offset."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import norm_cases as K  # noqa: E402

pytestmark = pytest.mark.gpu

BN_SHAPES = [(C, M) for C in (4, 8, 72, 216, 508, 512) for M in (4095, 4096, 4097, 70400)] + \
            [(C, M) for C in (516, 576, 1512, 2048) for M in (1, 7, 9, 1100, 4096)]
BN_CASES = [(C, M, shift, K.BN_VARIANTS[i % 4]) for i, (C, M) in enumerate(BN_SHAPES) for shift in (0.0, 10.0, 30.0)]
STATS_CASES = [(C, HW, nb) for C in (72, 512, 516, 1512, 2048) for HW in (1, 1023, 1024, 1760) for nb in (1, 3, 10)]
SE_CASES = [(C, hw) for hw in (1, 3, 110, 1024, 1760) for C in (72, 216, 576, 1512)]
LN_WIDTHS = [72, 216, 576, 1512, 1, 31, 257, 2049]


@pytest.fixture(scope='module')
def ctx():
    from transfuser_b200 import _lib
    return K.Ctx(_lib.call, 'cuda', torch.cuda.get_device_properties(0).multi_processor_count)


@pytest.fixture(scope='module')
def bench_rows():
    """The largest M that tfb_colsum and tfb_grad_prep see in one training step of the benchmarked configuration (TransFuser,
    batch 10, bf16), found by spying on the C-ABI calls of an eager step."""
    import numpy as np
    from bench import make_host_batch
    from test_tc_exact import _spy
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    torch.manual_seed(0)
    tr = Trainer(TrainConfig(), 'cuda', gemm_mode='bf16', lr=1e-4, seed=0, backbone='transFuser', raw_inputs=True)
    host = make_host_batch(10, seed=100, torch=torch, np=np, backbone='transFuser', raw=True)
    dev = {k: v.cuda() for k, v in host.items()}
    _, calls = _spy(lambda: tr.step(dev))
    torch.cuda.synchronize()
    rows = {'colsum': [(a[2], a[3]) for n, a in calls if n == 'tfb_colsum'],
            'grad_prep': [(a[6], a[7]) for n, a in calls if n == 'tfb_grad_prep']}
    del tr
    torch.cuda.empty_cache()
    assert rows['colsum'] and rows['grad_prep']
    print('bench step: colsum (M, C) max %s of %d calls; grad_prep (M, C) max %s of %d calls'
          % (max(rows['colsum']), len(rows['colsum']), max(rows['grad_prep']), len(rows['grad_prep'])))
    return {k: max(v) for k, v in rows.items()}


def _show(what, res):
    print('%s: %s' % (what, {k: '%.4f' % v if 'rel err' not in k else '%.2e' % v for k, v in res.items()}))


def _fresh(ctx):
    ctx.res = {}
    return ctx


@pytest.mark.parametrize('C,M,shift,variant', BN_CASES)
def test_bn_train_exact(ctx, C, M, shift, variant):
    _show('bn C %d M %d shift %g %s' % (C, M, shift, variant), K.bn_train(_fresh(ctx), C, M, shift, variant))


@pytest.mark.parametrize('C,HW,nb', STATS_CASES)
def test_bn_fwd_stats_exact(ctx, C, HW, nb):
    i = STATS_CASES.index((C, HW, nb))
    for variant in ('pool', K.STATS_VARIANTS[i % 3]):
        _show('bn_fwd_stats C %d HW %d x %d %s' % (C, HW, nb, variant), K.bn_fwd_stats(_fresh(ctx), C, HW, nb, variant))
    _show('bn_fwd pool C %d HW %d x %d' % (C, HW, nb), K.bn_fwd_pool(_fresh(ctx), C, HW, nb))


@pytest.mark.parametrize('C,hw', SE_CASES)
def test_bn_bwd_se_exact(ctx, C, hw):
    nb = -(-4100 // hw) if C <= 512 else 3            # narrow maps past M = 4096 (the flat reduction), wide ones a few samples
    _show('bn_bwd_se C %d hw %d x %d' % (C, hw, nb), K.bn_bwd_se(_fresh(ctx), C, hw, nb, side=SE_CASES.index((C, hw)) % 2 == 1))


@pytest.mark.parametrize('variant', ['relu', 'residual', 'y16'])
@pytest.mark.parametrize('C', [72, 516, 1512])
def test_bn_apply_exact(ctx, C, variant):
    _show('bn_apply C %d %s' % (C, variant), K.bn_apply(_fresh(ctx), C, 4099, variant))


@pytest.mark.parametrize('layout', K.COLSUM_LAYOUTS)
@pytest.mark.parametrize('C', [1, 3, 7, 12, 64, 648])
def test_colsum_exact(ctx, bench_rows, C, layout):
    for M in (1, 4095, 4096, bench_rows['colsum'][0]):
        _show('colsum C %d M %d %s' % (C, M, layout), K.colsum(_fresh(ctx), C, M, layout))


@pytest.mark.parametrize('relu', [True, False])
@pytest.mark.parametrize('C', [1, 7, 32, 216, 648, 4536])
def test_grad_prep_exact(ctx, bench_rows, C, relu):
    big = bench_rows['grad_prep'][0]                     # (its own width is 32; wider maps of that height do not fit with the fp64 references)
    for M in (1, 1740) + ((big,) if big * C <= 1 << 28 else ()):
        for outs in K.GRAD_PREP_OUTS:
            _show('grad_prep C %d M %d %s relu %d' % (C, M, outs, relu), K.grad_prep(_fresh(ctx), C, M, outs, relu))


@pytest.mark.parametrize('R', [1, 174, 1740])
@pytest.mark.parametrize('C', LN_WIDTHS)
def test_layernorm_exact(ctx, C, R):
    for acc in (False, True):
        _show('layernorm C %d R %d acc %d' % (C, R, acc), K.layernorm(_fresh(ctx), C, R, acc))


@pytest.mark.parametrize('p', [0.0, 0.1])
@pytest.mark.parametrize('C', LN_WIDTHS)
def test_add_dropout_ln_exact(ctx, C, p):
    for R, gx in ((1, False), (174, True), (1740, False)):
        _show('add_dropout_ln C %d R %d p %g gx %d' % (C, R, p, gx), K.add_dropout_ln(_fresh(ctx), C, R, p, gx))


def test_stream_reuse_exact(ctx):
    K.stream_reuse(ctx, [(K.bn_train, (72, 70400, 10.0, 'relu')), (K.colsum, (7, 4097, 'padded')), (K.layernorm, (257, 174, False)),
                         (K.bn_bwd_se, (576, 110, 3)), (K.grad_prep, (648, 1740, ('dbias',), True)), (K.bn_train, (1512, 1100, 0.0, 'residual')),
                         (K.bn_fwd_stats, (72, 1760, 10, 'pool')), (K.bn_fwd_pool, (516, 3, 10)), (K.add_dropout_ln, (1512, 174, 0.1, True)),
                         (K.bn_train, (8, 4097, 30.0, 'y16'))])


def test_misaligned_operands_refused(ctx):
    """Refused on the host: no misaligned operand is ever launched."""
    K.refusals(ctx)
