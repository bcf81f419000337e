"""The tensor-core PARITY modes ('bf16x3' / 'bf16x6', transfuser_b200/gemm.py): every fp32 operand is split into two / three bf16 terms
and each product runs as three / six tensor-core bf16 GEMMs (smallest terms first, fp32 accumulate). Held to the fp32 tolerance of test_ops.py — 1e-4
relative L2 per op against plain fp32 torch (north_star: 1e-3) — forward and backward, for every op the mode moves to the tensor cores:
nn.Linear / 1x1 convs (incl. stride 2), dense 3x3 convs (im2col + GEMM: forward, dgrad with flipped weights, wgrad) and the
attention projections. The whole-model parity test (tests/test_model.py) runs in this mode as well."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOL = 1e-4


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


NPROD = {'bf16x3': 3, 'bf16x6': 6}      # tensor-core GEMMs per fp32 product


@pytest.fixture(autouse=True, params=['bf16x3', 'bf16x6'])
def x3_mode(request):
    from transfuser_b200 import gemm
    old = gemm.MODE
    gemm.set_mode(request.param)
    yield request.param
    gemm.set_mode(old)


def _calls(fn):
    """Entry points fn() reaches (names), to check the products really run on the tensor-core kernel."""
    from transfuser_b200 import _lib
    L = _lib.lib()
    seen = []
    orig = L.call

    def spy(name, *a):
        seen.append(name)
        return orig(name, *a)

    L.call = spy
    try:
        out = fn()
    finally:
        del L.call
    return out, seen


def test_split_is_exact_to_two_bf16_terms(x3_mode):
    from transfuser_b200 import gemm
    x = rnd(37, 40, seed=1) * torch.logspace(-6, 6, 40, device=DEV)
    v = x[:, 4:36]                                  # strided view
    t = gemm.split_bf16(v)
    assert len(t) == (2 if x3_mode == 'bf16x3' else 3)
    assert all(a.dtype == torch.bfloat16 and a.is_contiguous() and a.shape == (37, 32) for a in t)
    assert torch.equal(t[0], v.to(torch.bfloat16))
    assert torch.equal(t[1], (v - t[0].float()).to(torch.bfloat16))
    assert rel(t[0].float() + t[1].float(), v) < 2 ** -16
    if len(t) == 3:
        assert torch.equal(t[2], (v - t[0].float() - t[1].float()).to(torch.bfloat16))
        assert torch.equal(t[0].double() + t[1].double() + t[2].double(), v.double())       # 3 x 8 bits: all 24 mantissa bits


@pytest.mark.parametrize('M,K,N', [(348, 72, 72), (348, 216, 864), (1740, 576, 576), (4096 + 64, 64, 16)])
def test_linear_x3_fwd_bwd(M, K, N, x3_mode):
    from transfuser_b200 import ops
    x, w, b = rnd(M, K, seed=1).requires_grad_(), rnd(N, K, seed=2, scale=1 / math.sqrt(K)).requires_grad_(), rnd(N, seed=3).requires_grad_()
    xm, wm, bm = [t.detach().clone().requires_grad_() for t in (x, w, b)]
    ref = F.relu(F.linear(x, w, b))
    out, seen = _calls(lambda: ops.linear(xm, wm, bm, relu=True))
    assert seen.count('tfb_gemm_bf16_tc') == NPROD[x3_mode] and 'tfb_gemm_f32_simt' not in seen
    assert rel(out, ref) < TOL
    # gradients without the ReLU: a pre-activation within rounding of 0 takes the other branch, a property of the comparison
    ref, out = F.linear(x, w, b), ops.linear(xm, wm, bm)
    assert rel(out, ref) < TOL
    go = rnd(M, N, seed=4)
    got, seen = _calls(lambda: torch.autograd.grad(out, [xm, wm, bm], go))
    assert seen.count('tfb_gemm_bf16_tc') == 2 * NPROD[x3_mode] and 'tfb_gemm_f32_simt' not in seen and 'tfb_conv2d_wgrad' not in seen
    for a, r in zip(got, torch.autograd.grad(ref, [x, w, b], go)):
        assert rel(a, r) < TOL


@pytest.mark.parametrize('cfg', [(2, 16, 24, 64, 64, 3, 1, True), (2, 10, 12, 512, 128, 3, 1, False), (3, 20, 16, 32, 32, 3, 1, True),
                                 (2, 20, 24, 72, 216, 1, 2, False), (2, 12, 16, 216, 216, 1, 1, False)])
def test_conv_x3_fwd_bwd(cfg, x3_mode):
    """Dense 3x3 (bias + ReLU as in the heads / decoders) and 1x1 (stride 1 and 2) convs, NHWC product vs NCHW torch."""
    from transfuser_b200 import ops
    N, H, W, Cin, Cout, ks, stride, bias = cfg
    x = rnd(N, Cin, H, W, seed=1).requires_grad_()
    w = rnd(Cout, Cin, ks, ks, seed=2, scale=1 / math.sqrt(Cin * ks * ks)).requires_grad_()
    b = rnd(Cout, seed=3).requires_grad_() if bias else None
    ref = F.conv2d(x, w, b, stride=stride, padding=ks // 2)
    if bias:
        ref = F.relu(ref)
    xm = x.detach().permute(0, 2, 3, 1).contiguous().requires_grad_()
    wm = w.detach().clone().requires_grad_()
    bm = b.detach().clone().requires_grad_() if bias else None
    out, seen = _calls(lambda: ops.conv2d(xm, wm, bm, stride=stride, relu=bias))
    assert seen.count('tfb_gemm_bf16_tc') == NPROD[x3_mode] and 'tfb_conv2d_fwd' not in seen
    assert rel(out.permute(0, 3, 1, 2), ref) < TOL
    if bias:      # gradients through the product's own ReLU mask (a pre-activation within rounding of 0 may take the other branch)
        ref = F.conv2d(x, w, b, stride=stride, padding=ks // 2) * (out.detach().permute(0, 3, 1, 2) > 0)
    go = rnd(*ref.shape, seed=4)
    ps, pr = [xm, wm] + ([bm] if bias else []), [x, w] + ([b] if bias else [])
    got, seen = _calls(lambda: torch.autograd.grad(out, ps, go.permute(0, 2, 3, 1).contiguous()))
    assert seen.count('tfb_gemm_bf16_tc') == 2 * NPROD[x3_mode] and 'tfb_conv2d_dgrad' not in seen and 'tfb_conv2d_wgrad' not in seen
    want = torch.autograd.grad(ref, pr, go)
    assert rel(got[0].permute(0, 3, 1, 2), want[0]) < TOL
    for a, r in zip(got[1:], want[1:]):
        assert rel(a, r) < TOL


def test_grouped_and_narrow_convs_stay_exact():
    """Grouped 3x3 (24 channels per group), the 3-channel stem and < 16-channel outputs run on the exact fp32 direct kernels."""
    from transfuser_b200 import ops
    for (Cin, Cout, groups) in ((72, 72, 3), (3, 32, 1), (32, 7, 1)):
        x = rnd(2, 12, 16, Cin, seed=1)
        w = rnd(Cout, Cin // groups, 3, 3, seed=2, scale=0.1)
        out, seen = _calls(lambda: ops.conv2d(x, w, None, stride=1, groups=groups))
        assert 'tfb_conv2d_fwd' in seen and 'tfb_gemm_bf16_tc' not in seen
        ref = F.conv2d(x.permute(0, 3, 1, 2), w, None, padding=1, groups=groups)
        assert rel(out.permute(0, 3, 1, 2), ref) < TOL


def test_attention_x3():
    from transfuser_b200 import ops
    B, T, C, nh = 2, 46, 216, 4
    h = rnd(B * T, C, seed=1).requires_grad_()
    ws = [rnd(C, C, seed=10 + i, scale=1 / math.sqrt(C)).requires_grad_() for i in range(3)]
    bs = [rnd(C, seed=20 + i, scale=0.1).requires_grad_() for i in range(3)]
    q, k, v = [F.linear(h, ws[i], bs[i]).view(B, T, nh, C // nh).transpose(1, 2) for i in range(3)]
    att = F.softmax((q @ k.transpose(-2, -1)) * (1.0 / math.sqrt(C // nh)), dim=-1)
    ref = (att @ v).transpose(1, 2).reshape(B * T, C)
    hm = h.detach().clone().requires_grad_()
    wm = [w.detach().clone().requires_grad_() for w in ws]
    bm = [b.detach().clone().requires_grad_() for b in bs]
    out, seen = _calls(lambda: ops.AttentionFn.apply(hm, wm[0], bm[0], wm[1], bm[1], wm[2], bm[2], B, T, nh, 0.0, 0))
    assert 'tfb_gemm_bf16_tc' in seen
    assert rel(out, ref) < TOL
    go = rnd(B * T, C, seed=5)
    got = torch.autograd.grad(out, [hm] + wm, go)
    want = torch.autograd.grad(ref, [h] + ws, go)
    for a, r in zip(got, want):
        assert rel(a, r) < TOL
