"""The elementwise, upsample and squeeze-excite kernels of csrc/elementwise.cu on the H100 at full size, against the float64
references of tests/elementwise_ref.py (cases: tests/elementwise_cases.py; the same cases at reduced size under the CPU emulation:
tests/test_elementwise_emulated.py). The shapes include those of every call site in a benchmark step (TransFuser, RegNetY-032,
batch 10): the decoder and FPN upsamples, the BEV head, the SE widths 72 / 216 / 576 / 1512 on the image and LiDAR maps, the GPT
grids 5x22 and 8x8 with their token build and attention softmax. Every case runs twice into NaN-filled, sentinel-guarded outputs
and must give the same bits. Each test prints its worst allowance ratio per check (1.0 = at the bound)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import elementwise_cases as K  # noqa: E402
import elementwise_ref as R  # noqa: E402
from test_elementwise_emulated import (EMUL_GPT, EMUL_POOL, EMUL_SE_MLP, EMUL_SE_REDUCE, EMUL_SE_SCALE, EMUL_TOKENS,  # noqa: E402
                                       EMUL_UPSAMPLE, EMUL_WINDOWS)

pytestmark = pytest.mark.gpu

# image maps of the stages: 40x176 (72), 20x88 (216), 10x44 (576), 5x22 (1512); LiDAR: 64x64, 32x32, 16x16, 8x8
IMG = [(40, 176, 72), (20, 88, 216), (10, 44, 576), (5, 22, 1512)]
LID = [(64, 64, 72), (32, 32, 216), (16, 16, 576), (8, 8, 1512)]
# (N, Hi, Wi, Ho, Wo, C, align_corners, sidecar): decoder / FPN x2 steps at C = 64, the decoder's last x4, the BEV head to 160x160
UPSAMPLE = [(10, 5, 22, 10, 44, 64, 0, True), (10, 10, 44, 20, 88, 64, 0, True), (10, 20, 88, 40, 176, 64, 0, True),
            (2, 40, 176, 160, 704, 64, 0, True), (10, 8, 8, 16, 16, 64, 0, True), (10, 16, 16, 32, 32, 64, 0, True),
            (10, 32, 32, 64, 64, 64, 0, True), (10, 64, 64, 160, 160, 3, 1, False), (10, 64, 64, 160, 160, 4, 1, False)]


@pytest.fixture(scope='module')
def ctx():
    from transfuser_b200 import _lib
    return K.Ctx(_lib.call, 'cuda', torch.cuda.get_device_properties(0).multi_processor_count)


def _show(what, res):
    print('%s: %s' % (what, {k: '%.4f' % v for k, v in res.items()}))


def _fresh(ctx):
    ctx.res = {}
    return ctx


@pytest.mark.parametrize('N,Hi,Wi,Ho,Wo,C,ac,side', UPSAMPLE + EMUL_UPSAMPLE + EMUL_WINDOWS)
def test_upsample_exact(ctx, N, Hi, Wi, Ho, Wo, C, ac, side):
    _show('upsample %dx%d -> %dx%d C %d ac %d (window %d)' % (Hi, Wi, Ho, Wo, C, ac, R.max_window(Wi, Wo, ac)),
          K.upsample(_fresh(ctx), N, Hi, Wi, Ho, Wo, C, ac, side))


@pytest.mark.parametrize('N,H,W,C,gh,gw,side', [(10, H, W, C, 5, 22, True) for H, W, C in IMG] + [(10, H, W, C, 8, 8, True) for H, W, C in LID]
                         + [(10, 40, 176, 70, 5, 22, False)] + EMUL_GPT)
def test_gpt_up_add_exact(ctx, N, H, W, C, gh, gw, side):
    _show('gpt_up_add %dx%d C %d grid %dx%d' % (H, W, C, gh, gw), K.gpt_up_add(_fresh(ctx), N, H, W, C, gh, gw, side))


SE_MAPS = [(10, H * W, C) for H, W, C in IMG + LID]


@pytest.mark.parametrize('N,HW,C', SE_MAPS + [(10, 1, 1512), (1, 8200, 4), (3, 300000, 8)] + EMUL_POOL)
def test_pool_hw_exact(ctx, N, HW, C):
    _show('pool_hw N %d HW %d C %d' % (N, HW, C), K.pool_hw(_fresh(ctx), N, HW, C))


@pytest.mark.parametrize('N,HW,C', SE_MAPS + [(10, 1023, 72), (10, 1024, 72), (10, 1025, 216), (64, 4096, 72), (200, 8192, 8)]
                         + EMUL_SE_REDUCE)
def test_se_reduce_exact(ctx, N, HW, C):
    _show('se_reduce N %d HW %d C %d' % (N, HW, C), K.se_reduce(_fresh(ctx), N, HW, C))


@pytest.mark.parametrize('N,HW,C,side', [(N, HW, C, True) for N, HW, C in SE_MAPS] + [(10, 1760, 70, True)] + EMUL_SE_SCALE)
def test_se_scale_exact(ctx, N, HW, C, side):
    _show('se_scale N %d HW %d C %d' % (N, HW, C), K.se_scale(_fresh(ctx), N, HW, C, side))


@pytest.mark.parametrize('N,C,Cr', [(10, 72, 8), (10, 216, 18), (10, 216, 54), (10, 576, 54), (10, 576, 144), (10, 1512, 144), (16, 1512, 378),
                                    (16, 2000, 512)] + EMUL_SE_MLP)
def test_se_mlp_bwd_exact(ctx, N, C, Cr):
    _show('se_mlp_bwd N %d C %d Cr %d' % (N, C, Cr), K.se_mlp_bwd(_fresh(ctx), N, C, Cr))


@pytest.mark.parametrize('N,C,img_hw,img_grid,lid_hw,lid_grid', [(10, C, (H, W), (5, 22), LID[i][:2], (8, 8)) for i, (H, W, C) in enumerate(IMG)]
                         + EMUL_TOKENS)
def test_tokens_exact(ctx, N, C, img_hw, img_grid, lid_hw, lid_grid):
    _show('tokens C %d %s %s' % (C, img_hw, lid_hw), K.tokens(_fresh(ctx), N, C, img_hw, img_grid, lid_hw, lid_grid))


@pytest.mark.parametrize('N,A,B', [(10, 174, 72), (10, 1512, 174), (2, 33, 45), (1, 1, 70), (3, 64, 31), (1, 100, 1), (40, 1000, 999)])
def test_transpose_exact(ctx, N, A, B):
    K.transpose(_fresh(ctx), N, A, B)


@pytest.mark.parametrize('N,H,W', [(10, 160, 704), (2, 5, 7)])
def test_image_prep_exact(ctx, N, H, W):
    K.image_prep(_fresh(ctx), N, H, W)


@pytest.mark.parametrize('n,relu,side', [(1, True, False), (7, True, True), (1030, True, True), (4099, False, True),
                                         (10 * 40 * 176 * 72 + 3, True, True), (10 * 8 * 8 * 1512, False, False)])
def test_add_relu_exact(ctx, n, relu, side):
    K.add_relu(_fresh(ctx), n, relu, side)


@pytest.mark.parametrize('n', [13, 1000, 10 * 1512 + 1, 1 << 22])
def test_activations_exact(ctx, n):
    _show('activations n %d' % n, K.activations(_fresh(ctx), n))


@pytest.mark.parametrize('N,H,W,C', [(10, 40, 176, 72), (10, 20, 88, 216), (10, 11, 45, 576), (10, 9, 9, 1512), (2, 7, 9, 4), (1, 5, 5, 3),
                                     (2, 6, 8, 8), (1, 1, 1, 4)])
def test_stride2_exact(ctx, N, H, W, C):
    K.stride2(_fresh(ctx), N, H, W, C)


@pytest.mark.parametrize('N,T,C', [(10, 174, 72), (10, 174, 1512), (2, 3, 5)])
def test_scale_bcast_exact(ctx, N, T, C):
    _show('scale_dev / bcast_add N %d T %d C %d' % (N, T, C), K.scale_bcast(_fresh(ctx), N, T, C))


@pytest.mark.parametrize('rows,L', [(10 * 4 * 174, 174), (9, 7), (100, 31), (100, 32), (100, 33), (64, 1000)])
def test_softmax_exact(ctx, rows, L):
    _show('softmax rows %d L %d' % (rows, L), K.softmax(_fresh(ctx), rows, L))


def test_misaligned_operands_refused(ctx):
    """Refused on the host: no misaligned operand is ever launched. (The scalar fallbacks are checked under the emulation.)"""
    K.misaligned(ctx, fallbacks=False)
