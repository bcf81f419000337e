"""Float64 references and operand generators for the exact-fp32 CUDA-core kernels (csrc/conv_simt.cu, csrc/gemm_simt.cu).
Plain torch, no product imports.

Two kinds of operands:
- exact: small integers times a power of two. When K * max|a| * max|b| (plus the epilogue terms) stays below 2^24 units of the
  finest grid any term lies on, every partial sum of every order is exact in fp32, so the kernel must equal the float64 result
  bit for bit (assert_exact checks the condition for each case). One dropped, doubled or misplaced term shows up in full.
- Gaussian, plain or mean-shifted (cancelling sums): element by element within K * 2^-23 * (|a| |b|), K the number of terms of that
  output, which bounds every summation tree, plus 2^-23 * |v| for each rounding of the epilogue.
"""
import math

import torch
import torch.nn.functional as F

EPS32 = 2.0 ** -23
LIMIT = 2 ** 24


# ------------------------------------------------------------------ operands
def dyadic(shape, r, e, seed, device):
    """Integers in [-r, r] times 2^-e (exact in fp32)."""
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randint(-r, r + 1, shape, generator=g, device=device).float() * 2.0 ** -e


def gauss(shape, seed, device, scale=1.0, shift=0.0):
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randn(shape, generator=g, device=device) * scale + shift


def exact_range(K, r=8):
    """The largest power-of-two integer range r' <= r for both operands with K * r'^2 < 2^24 (one product is at most r'^2 units)."""
    while r > 1 and K * r * r >= LIMIT:
        r //= 2
    assert K < LIMIT, K
    return r


def assert_exact(K, amax, bmax, grid, extra=0.0, what=''):
    """K products of magnitude <= amax * bmax, plus `extra` (the magnitude of the epilogue terms), on a grid of spacing `grid`
    (the finest any term lies on): every partial sum fits 24 bits."""
    units = (K * amax * bmax + extra) / grid
    assert units < LIMIT, '%s: %d terms reach %.3g units of 2^%d, not exact in fp32' % (what, K, units, round(math.log2(grid)))


def bits_equal(out, ref, what):
    """out (fp32) equals the float64 value ref exactly everywhere (the sign of a zero aside)."""
    o = out.double()
    assert bool(torch.isfinite(o).all()), '%s: %d non-finite elements' % (what, int((~torch.isfinite(o)).sum()))
    assert bool((ref.float().double() == ref).all()), '%s: the exact reference is not representable in fp32' % what
    ne = o != ref
    if bool(ne.any()):
        i = tuple(int(v) for v in ne.nonzero()[0])
        raise AssertionError('%s: %d of %d elements differ from the exact result, first at %s: %.9g, exact %.9g'
                             % (what, int(ne.sum()), ne.numel(), i, o[i].item(), ref[i].item()))


# ------------------------------------------------------------------ convolutions (NHWC activations, [Cout][Cin/g][k][k] weights)
def out_hw(H, W, k, stride):
    p = k // 2
    return (H + 2 * p - k) // stride + 1, (W + 2 * p - k) // stride + 1


def _nchw(t):
    return t.double().permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def conv_fwd(x, w, bias, stride, groups, relu):
    """(y, |x| * |w| + |bias|) in fp64, NHWC."""
    k = w.shape[2]
    y = F.conv2d(_nchw(x), w.double(), None, stride, k // 2, 1, groups)
    mag = F.conv2d(_nchw(x).abs(), w.double().abs(), None, stride, k // 2, 1, groups)
    if bias is not None:
        y = y + bias.double().view(1, -1, 1, 1)
        mag = mag + bias.double().abs().view(1, -1, 1, 1)
    if relu:
        y = y.clamp_min(0)
    return _nhwc(y), _nhwc(mag)


def conv_dgrad(dy, w, x_shape, stride, groups):
    """(dx, |dy| * |w|) in fp64, NHWC."""
    N, H, W, Cin = x_shape
    k = w.shape[2]
    shp = (N, Cin, H, W)
    dx = torch.nn.grad.conv2d_input(shp, w.double(), _nchw(dy), stride, k // 2, 1, groups)
    mag = torch.nn.grad.conv2d_input(shp, w.double().abs(), _nchw(dy).abs(), stride, k // 2, 1, groups)
    return _nhwc(dx), _nhwc(mag)


def conv_wgrad(x, dy, w_shape, stride, groups):
    """(dw, |x| * |dy|, dbias, sum |dy|) in fp64."""
    k = w_shape[2]
    xd, gd = _nchw(x), _nchw(dy)
    dw = torch.nn.grad.conv2d_weight(xd, w_shape, gd, stride, k // 2, 1, groups)
    mag = torch.nn.grad.conv2d_weight(xd.abs(), w_shape, gd.abs(), stride, k // 2, 1, groups)
    return dw, mag, gd.sum((0, 2, 3)), gd.abs().sum((0, 2, 3))


# ------------------------------------------------------------------ GEMMs
def op(t, trans):
    t = t.double()
    return t.transpose(-1, -2) if trans else t


def gemm(A, B, ta, tb, alpha, beta, C0, bias, relu):
    """alpha * op(A) @ op(B) (+ bias[n]) (+ beta * C0) (ReLU), and its magnitude, in fp64. A, B, C0: [..., rows, cols] as stored."""
    a, b = op(A, ta), op(B, tb)
    v, mag = alpha * (a @ b), abs(alpha) * (a.abs() @ b.abs())
    if bias is not None:
        v, mag = v + bias.double(), mag + bias.double().abs()
    if beta != 0:
        v, mag = v + beta * C0.double(), mag + abs(beta) * C0.double().abs()
    if relu:
        v = v.clamp_min(0)
    return v, mag


def small_m(A, B, tb, bias):
    """The pre-activation A @ op(B) (+ bias) and its magnitude, fp64."""
    return gemm(A, B, False, bool(tb), 1.0, 0.0, None, bias, False)


def sigmoid(v):
    return 1.0 / (1.0 + torch.exp(-v.double()))


def sigmoid_allow(v, v_err):
    """Allowance of the kernel's 1 / (1 + expf(-v)) against fp64 sigmoid(v): expf within 2 ulp (CUDA's bound), the rounding of
    1 + e and of the division (a relative error of at most 4 * 2^-23 in all), plus the error v_err of the pre-activation itself
    through the slope s (1 - s)."""
    s = sigmoid(v)
    return 4 * EPS32 * s + s * (1 - s) * v_err + 2.0 ** -149
