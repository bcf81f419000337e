"""The elementwise, upsample and squeeze-excite kernels of csrc/elementwise.cu under the CPU emulation (2 SMs), at reduced sizes that
still cross every dispatch boundary: the float4 and scalar forms, the bilinear gather windows under, at and over GATHER_W = 24 pixels
with and without align_corners, the pooling split counts 1 .. 32, the flat and slab squeeze-excite reductions (HW around 1024, the
4 * SMs / N split cap), the scalar tails. Cases: tests/elementwise_cases.py; on the H100 at full size: tests/test_elementwise_exact.py."""
import pytest

import elementwise_cases as K
import elementwise_ref as R
from cuda_emul import loader

SMS = 2
# (N, Hi, Wi, Ho, Wo, C, align_corners, bf16 sidecar)
EMUL_UPSAMPLE = [(2, 5, 11, 20, 44, 4, 0, True), (2, 5, 11, 20, 44, 6, 0, True), (2, 7, 5, 19, 23, 8, 0, False),
                 (2, 7, 5, 19, 23, 3, 1, True), (2, 7, 5, 19, 23, 4, 1, False), (1, 6, 6, 6, 6, 4, 1, False), (1, 6, 6, 6, 6, 3, 0, False),
                 (2, 9, 9, 4, 5, 4, 0, False), (2, 9, 9, 4, 5, 5, 1, False), (1, 3, 1, 7, 9, 4, 1, False), (1, 3, 1, 7, 9, 3, 0, False),
                 (1, 1, 3, 9, 7, 4, 0, True), (1, 4, 4, 1, 1, 4, 1, False), (1, 4, 5, 3, 1, 3, 0, False), (1, 16, 16, 40, 40, 3, 1, False),
                 (1, 16, 16, 40, 40, 4, 1, True)]
# gather windows (lerp_window, in destination pixels) just under, at and over GATHER_W, for both forms and both align_corners
EMUL_WINDOWS = [(1, s, s, o, o, C, ac, False) for s, o, ac in ((3, 29, 0), (3, 30, 0), (3, 31, 0), (4, 38, 0), (4, 39, 0),
                                                               (3, 23, 1), (3, 24, 1), (3, 25, 1), (3, 28, 1), (4, 29, 1), (4, 30, 1))
                for C in (4, 3)]
# (N, H, W, C, gh, gw, sidecar)
EMUL_GPT = [(2, 10, 44, 8, 5, 22, True), (2, 10, 44, 6, 5, 22, False), (2, 16, 16, 4, 8, 8, True), (1, 7, 9, 3, 8, 8, False),
            (1, 40, 40, 4, 2, 2, False)]
EMUL_POOL = [(2, 7, 8), (2, 300, 8), (3, 1100, 12), (1, 8200, 4), (2, 300, 72), (1, 40, 1512)]
EMUL_SE_REDUCE = [(2, 1023, 72), (2, 1024, 72), (2, 1025, 72), (2, 4096, 72), (9, 1024, 8), (2, 300, 216), (1, 40, 1512), (3, 2000, 576)]
EMUL_SE_SCALE = [(2, 7, 72, True), (2, 7, 6, True), (2, 5, 1512, False), (1, 3, 5, False)]
EMUL_SE_MLP = [(1, 72, 3), (16, 72, 8), (16, 216, 18), (4, 576, 54), (16, 1512, 144), (2, 100, 7), (3, 40, 512)]
EMUL_TOKENS = [(2, 8, (10, 44), (5, 22), (16, 16), (8, 8)), (1, 5, (5, 22), (5, 22), (8, 8), (8, 8)), (2, 4, (20, 44), (5, 22), (24, 8), (8, 8))]


@pytest.fixture(scope='module')
def ctx():
    return K.Ctx(loader.emul().call, 'cpu', SMS)


def _show(what, res):
    print('%s: %s' % (what, {k: '%.4f' % v for k, v in res.items()}))


def _fresh(ctx):
    ctx.res = {}
    return ctx


@pytest.mark.parametrize('N,Hi,Wi,Ho,Wo,C,ac,side', EMUL_UPSAMPLE + EMUL_WINDOWS)
def test_upsample_emulated(ctx, N, Hi, Wi, Ho, Wo, C, ac, side):
    _show('upsample %dx%d -> %dx%d C %d ac %d (window %d)' % (Hi, Wi, Ho, Wo, C, ac, R.max_window(Wi, Wo, ac)),
          K.upsample(_fresh(ctx), N, Hi, Wi, Ho, Wo, C, ac, side))


def test_window_cases_cross_gather_w():
    """The window cases reach widths under, at and over GATHER_W with each align_corners setting."""
    for ac in (0, 1):
        w = {R.max_window(s, o, a) for _, s, _, o, _, _, a, _ in EMUL_WINDOWS if a == ac}
        assert {R.GATHER_W - 1, R.GATHER_W, R.GATHER_W + 1} <= w, (ac, sorted(w))


@pytest.mark.parametrize('N,H,W,C,gh,gw,side', EMUL_GPT)
def test_gpt_up_add_emulated(ctx, N, H, W, C, gh, gw, side):
    _show('gpt_up_add %dx%d C %d grid %dx%d' % (H, W, C, gh, gw), K.gpt_up_add(_fresh(ctx), N, H, W, C, gh, gw, side))


@pytest.mark.parametrize('N,HW,C', EMUL_POOL)
def test_pool_hw_emulated(ctx, N, HW, C):
    _show('pool_hw N %d HW %d C %d' % (N, HW, C), K.pool_hw(_fresh(ctx), N, HW, C))


@pytest.mark.parametrize('N,HW,C', EMUL_SE_REDUCE)
def test_se_reduce_emulated(ctx, N, HW, C):
    _show('se_reduce N %d HW %d C %d' % (N, HW, C), K.se_reduce(_fresh(ctx), N, HW, C))


@pytest.mark.parametrize('N,HW,C,side', EMUL_SE_SCALE)
def test_se_scale_emulated(ctx, N, HW, C, side):
    _show('se_scale N %d HW %d C %d' % (N, HW, C), K.se_scale(_fresh(ctx), N, HW, C, side))


@pytest.mark.parametrize('N,C,Cr', EMUL_SE_MLP)
def test_se_mlp_bwd_emulated(ctx, N, C, Cr):
    _show('se_mlp_bwd N %d C %d Cr %d' % (N, C, Cr), K.se_mlp_bwd(_fresh(ctx), N, C, Cr))


@pytest.mark.parametrize('N,C,img_hw,img_grid,lid_hw,lid_grid', EMUL_TOKENS)
def test_tokens_emulated(ctx, N, C, img_hw, img_grid, lid_hw, lid_grid):
    _show('tokens C %d %s %s' % (C, img_hw, lid_hw), K.tokens(_fresh(ctx), N, C, img_hw, img_grid, lid_hw, lid_grid))


@pytest.mark.parametrize('N,A,B', [(2, 33, 45), (1, 1, 70), (3, 64, 31), (1, 100, 1)])
def test_transpose_emulated(ctx, N, A, B):
    K.transpose(_fresh(ctx), N, A, B)


def test_image_prep_emulated(ctx):
    K.image_prep(_fresh(ctx), 2, 5, 7)


@pytest.mark.parametrize('n,relu,side', [(1, True, False), (7, True, True), (1030, True, True), (1030, False, False), (4099, False, True)])
def test_add_relu_emulated(ctx, n, relu, side):
    K.add_relu(_fresh(ctx), n, relu, side)


@pytest.mark.parametrize('n', [13, 1000])
def test_activations_emulated(ctx, n):
    _show('activations n %d' % n, K.activations(_fresh(ctx), n))


@pytest.mark.parametrize('N,H,W,C', [(2, 7, 9, 4), (1, 5, 5, 3), (2, 6, 8, 8), (1, 1, 1, 4)])
def test_stride2_emulated(ctx, N, H, W, C):
    K.stride2(_fresh(ctx), N, H, W, C)


@pytest.mark.parametrize('N,T,C', [(2, 3, 5), (3, 174, 8)])
def test_scale_bcast_emulated(ctx, N, T, C):
    _show('scale_dev / bcast_add N %d T %d C %d' % (N, T, C), K.scale_bcast(_fresh(ctx), N, T, C))


@pytest.mark.parametrize('rows,L', [(9, 7), (10, 32), (5, 33), (6, 174)])
def test_softmax_emulated(ctx, rows, L):
    _show('softmax rows %d L %d' % (rows, L), K.softmax(_fresh(ctx), rows, L))


def test_misaligned_operands_emulated(ctx):
    K.misaligned(ctx)
