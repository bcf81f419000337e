"""The ResNet stem kernels (csrc/resnet_stem.cu) executed unchanged on the CPU through the emulation in tests/cuda_emul/ (stem_emul.py), by their
C-ABI entry points: the 7x7 / stride-2 conv (forward, weight gradient) against fp64 F.conv2d within the fp32 accumulation bound,
and the 3x3 / stride-2 max-pool (forward, backward) bitwise against PyTorch's fp32 CPU max_pool2d. tests/test_resnet_gpu.py runs
the same checks on the device. Test infrastructure only."""
import pytest
import torch
import torch.nn.functional as F

from cuda_emul import stem_emul

U = 2.0 ** -23


def _call(name, *args):
    return stem_emul.call(name, *args)


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def stem_case(N, Cin, Cout, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 7, 7, generator=g) * 0.1
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    dy = torch.randn(N, Cout, Ho, Wo, generator=g)
    return x, w, dy


def check_stem(call, x, w, dy, to_dev=lambda t: t):
    """Forward and weight gradient of the 7x7 stem entry points against fp64 F.conv2d: every element within the worst-case fp32
    accumulation bound K * 2^-23 * (|x| |w|) of its K terms. The weight gradient gives the same bits on two calls."""
    N, Cin, H, W = x.shape
    Cout = w.shape[0]
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xd, wd, dyd = to_dev(_nhwc(x)), to_dev(w.contiguous()), to_dev(_nhwc(dy))
    y = to_dev(torch.full((N, Ho, Wo, Cout), float('nan')))
    call('tfb_conv7x7s2_fwd', xd, wd, y, N, H, W, Cin, Cout)
    want = F.conv2d(x.double(), w.double(), stride=2, padding=3)
    bound = Cin * 49 * U * F.conv2d(x.double().abs(), w.double().abs(), stride=2, padding=3)
    err = (y.cpu().double().permute(0, 3, 1, 2) - want).abs()
    assert bool((err <= bound + 1e-30).all()), float((err / bound.clamp_min(1e-30)).max())
    dws = []
    for _ in range(2):
        dw = to_dev(torch.full((Cout, Cin, 7, 7), float('nan')))
        call('tfb_conv7x7s2_wgrad', xd, dyd, dw, N, H, W, Cin, Cout)
        dws.append(dw.cpu())
    assert torch.equal(dws[0].view(torch.int32), dws[1].view(torch.int32))
    want = torch.nn.grad.conv2d_weight(x.double(), w.shape, dy.double(), stride=2, padding=3)
    bound = N * Ho * Wo * U * torch.nn.grad.conv2d_weight(x.double().abs(), w.shape, dy.double().abs(), stride=2, padding=3)
    err = (dws[0].double() - want).abs()
    assert bool((err <= bound + 1e-30).all()), float((err / bound.clamp_min(1e-30)).max())


def pool_case(N, C, H, W, seed):
    """Quantised values (many ties), a block of all-zero windows (as after BatchNorm + ReLU) and one NaN."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-3, 4, (N, C, H, W), generator=g).float().clamp_min(0) * 0.5
    x[:, :, :min(H, 4), :min(W, 6)] = 0.0
    x[0, C - 1, H // 2, W // 2] = float('nan')
    dy = torch.randn(N, C, (H - 1) // 2 + 1, (W - 1) // 2 + 1, generator=g)
    return x, dy


def bits(t):
    return t.contiguous().view(torch.int32)


def check_pool(call, x, dy, to_dev=lambda t: t):
    """Forward (fp32, its bf16 copy, the argmax tap) and backward bitwise against torch's fp32 CPU max_pool2d."""
    N, C, H, W = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xr = x.clone().requires_grad_()
    want, idx = F.max_pool2d(xr, 3, 2, 1, return_indices=True)
    want_dx, = torch.autograd.grad(want, xr, dy)
    xd, dyd = to_dev(_nhwc(x)), to_dev(_nhwc(dy))
    y = to_dev(torch.full((N, Ho, Wo, C), float('nan')))
    y16 = to_dev(torch.zeros((N, Ho, Wo, C), dtype=torch.bfloat16))
    arg = to_dev(torch.full((N, Ho, Wo, C), 255, dtype=torch.uint8))
    call('tfb_maxpool3x3s2_fwd', xd, y, y16, arg, N, H, W, C)
    assert torch.equal(bits(y.cpu().permute(0, 3, 1, 2)), bits(want.detach()))
    h, want16 = y16.cpu(), y.cpu().bfloat16()
    nan = want16.isnan()
    assert torch.equal(h.isnan(), nan) and torch.equal(h[~nan].view(torch.int16), want16[~nan].view(torch.int16))   # (NaN payloads differ)
    # the argmax tap names the element torch's index names
    ho = torch.arange(Ho).view(1, 1, Ho, 1)
    wo = torch.arange(Wo).view(1, 1, 1, Wo)
    a = arg.cpu().permute(0, 3, 1, 2).long()
    assert torch.equal((ho * 2 - 1 + a // 3) * W + (wo * 2 - 1 + a % 3), idx)
    dx = to_dev(torch.full((N, H, W, C), float('nan')))
    call('tfb_maxpool3x3s2_bwd', dyd, arg, dx, N, H, W, C)
    assert torch.equal(bits(dx.cpu().permute(0, 3, 1, 2)), bits(want_dx))
    return y, arg, dx


@pytest.mark.parametrize('N,Cin,Cout,H,W', [(2, 3, 64, 23, 30), (1, 2, 40, 16, 9), (2, 4, 32, 7, 7), (1, 1, 8, 12, 20)])
def test_stem_conv_emulated(N, Cin, Cout, H, W):
    check_stem(_call, *stem_case(N, Cin, Cout, H, W, seed=N * 100 + Cin * 10 + H))


@pytest.mark.parametrize('N,C,H,W', [(1, 4, 80, 352), (1, 8, 128, 128), (2, 8, 5, 7)])
def test_maxpool_emulated(N, C, H, W):
    check_pool(_call, *pool_case(N, C, H, W, seed=H + W))


def test_stem_and_pool_argument_checks():
    x = torch.zeros(1, 8, 8, 5)
    with pytest.raises(RuntimeError, match='argument check'):
        _call('tfb_conv7x7s2_fwd', x, torch.zeros(8, 5, 7, 7), torch.zeros(1, 4, 4, 8), 1, 8, 8, 5, 8)       # Cin > 4
    with pytest.raises(RuntimeError, match='argument check'):
        _call('tfb_maxpool3x3s2_fwd', torch.zeros(1, 8, 8, 6), torch.zeros(1, 4, 4, 6), None, torch.zeros(1, 4, 4, 6, dtype=torch.uint8),
              1, 8, 8, 6)                                                                                          # C % 4 != 0
