"""GEMM entry points of the C-ABI vs a plain fp32 torch reference of the same op (fp64-accumulated on the GPU)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [  # (M, N, K)
    (128, 64, 32), (128, 128, 256), (300, 72, 72), (1740, 1512, 1512), (174, 216, 864), (70400 // 8, 72, 24 * 3),
    (257, 200, 100), (64, 1512, 6048), (1, 64, 512), (20, 3, 64), (513, 576, 144),
]


def _ref(a, b, ta, tb, bias, relu, alpha, beta, c0):
    A = a.double().t() if ta else a.double()
    B = b.double().t() if tb else b.double()
    r = alpha * (A @ B)
    if bias is not None:
        r = r + bias.double()
    if beta != 0:
        r = r + beta * c0.double()
    if relu:
        r = r.clamp_min(0)
    return r


def _mk(M, N, K, ta, tb, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    a = torch.randn((K, M) if ta else (M, K), device='cuda', generator=g)
    b = torch.randn((N, K) if tb else (K, N), device='cuda', generator=g)
    return a, b


def _relerr(x, r):
    return ((x.double() - r).norm() / r.norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize('shape', SHAPES)
@pytest.mark.parametrize('ta,tb', [(False, True), (False, False), (True, False), (True, True)])
def test_simt_exact(shape, ta, tb):
    from transfuser_b200 import gemm
    M, N, K = shape
    a, b = _mk(M, N, K, ta, tb, 1)
    bias = torch.randn(N, device='cuda')
    c0 = torch.randn(M, N, device='cuda')
    out = c0.clone()
    gemm.gemm(a, b, out, ta, tb, bias=bias, relu=True, alpha=0.5, beta=1.0, mode='simt')
    assert _relerr(out, _ref(a, b, ta, tb, bias, True, 0.5, 1.0, c0)) < 1e-5


@pytest.mark.parametrize('shape', [s for s in SHAPES if s[1] >= 8 and s[2] >= 8])
@pytest.mark.parametrize('ta,tb', [(False, True), (False, False), (True, False), (True, True)])
def test_tf32_tensor_core(shape, ta, tb):
    """kind::tf32 keeps 10 mantissa bits of each operand: tolerance 2e-3 relative (||.||2), stated by north_star as 1e-3
    for fp32 — the SIMT path above is the fp32-exact mode; this bounds the tensor-core mode."""
    from transfuser_b200 import gemm
    M, N, K = shape
    if (M if ta else K) % 4 or (K if tb else N) % 4:
        pytest.skip('leading dimension not 16-byte aligned: served by the SIMT kernel')
    a, b = _mk(M, N, K, ta, tb, 2)
    bias = torch.randn(N, device='cuda')
    out = torch.full((M, N), float('nan'), device='cuda')
    gemm.gemm(a, b, out, ta, tb, bias=bias, relu=False, mode='tf32')
    assert _relerr(out, _ref(a, b, ta, tb, bias, False, 1.0, 0.0, None)) < 2e-3
    # split-K (wgrad shape class): per-split partial tiles added in split order
    out2 = torch.full((M, N), float('nan'), device='cuda')
    gemm.gemm(a, b, out2, ta, tb, bias=bias, splits=4, mode='tf32')
    assert _relerr(out2, _ref(a, b, ta, tb, bias, False, 1.0, 0.0, None)) < 2e-3


def test_strided_views_and_beta():
    from transfuser_b200 import gemm
    x = torch.randn(348, 3 * 216, device='cuda')
    w = torch.randn(216, 216, device='cuda')
    for mode in ('simt', 'tf32'):
        out = torch.zeros(348, 3 * 216, device='cuda')
        gemm.gemm(x[:, 216:432], w, out[:, 432:], False, True, mode=mode)
        r = x[:, 216:432].double() @ w.double().t()
        assert _relerr(out[:, 432:], r) < 2e-3
        assert out[:, :432].abs().sum().item() == 0
        acc = torch.ones(348, 216, device='cuda')
        gemm.gemm(x[:, :216], w, acc, False, True, beta=1.0, relu=True, mode=mode)
        assert _relerr(acc, (x[:, :216].double() @ w.double().t() + 1).clamp_min(0)) < 2e-3
