"""The im2col-free 3x3 weight gradient (tfb_conv3x3_tc_wgrad: the batched wgrad GEMM with its B tiles gathered from the activation)
against tfb_im2col3x3_bf16 + tfb_gemm_bf16_tc_wgrad_batched, which it must match bit for bit, and against the exact-operand reference
of tests/tc_ref.py (the same bf16 operands contracted in fp64, element by element at the worst-case fp32 accumulation bound). The
output is pre-filled with NaN (every element must be written) and followed by sentinels (nothing past dW is written); every case runs
twice and must give the same bits. Then one eager training step of the model with the gathered path on and off: the same bits.

The relative-L2 bound is 10x the worst value measured on an H100.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tc_ref as R  # noqa: E402
from tc_ref import Guarded  # noqa: E402
from test_tc_exact import _call  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda'
WGRAD_TOL = 8e-5         # 10x the measured worst relative L2 against the fp64 contraction, 7.7e-6 (the 160 x 704 decoder case)

CASES = [
    # N, H, W, Cin, Cout, ldg, groups, stride, splits (0: chosen by the library), grid cap (0: none)
    (2, 20, 36, 32, 32, 32, 1, 1, 0, 0),
    (2, 16, 40, 64, 64, 64, 1, 1, 0, 64),     # the weight-gradient stream's grid cap
    (1, 24, 40, 128, 128, 128, 1, 1, 3, 0),   # explicit split-K
    (2, 5, 22, 512, 64, 64, 1, 1, 0, 64),
    (1, 17, 33, 96, 40, 40, 1, 1, 0, 0),      # a partial 64-column chunk
    (2, 21, 35, 64, 256, 256, 1, 2, 0, 64),   # stride 2, two 128-row tiles
    (3, 23, 37, 32, 64, 64, 1, 2, 0, 0),      # stride 2, odd sizes
    (2, 33, 47, 72, 72, 72, 3, 1, 0, 64),     # grouped, odd group count
    (2, 29, 41, 216, 216, 216, 9, 2, 0, 64),  # grouped, stride 2
    (1, 6, 11, 1512, 1512, 1512, 63, 1, 0, 64),
    (2, 40, 70, 32, 7, 8, 1, 1, 0, 64),       # 7 output channels through zero-padded dy
    (2, 40, 70, 32, 1, 8, 1, 1, 0, 64),       # 1 output channel
    (2, 160, 704, 32, 32, 32, 1, 1, 0, 64),   # the full-size decoder conv
]


def _inputs(N, H, W, Cin, Cout, ldg, groups, stride):
    gen = torch.Generator(device=DEV).manual_seed(Cin * 7 + Cout + H)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    x = torch.randn(N, H, W, Cin, device=DEV, generator=gen)
    dy16 = torch.zeros(N, Ho, Wo, ldg, device=DEV, dtype=torch.bfloat16)
    dy16[..., :Cout] = torch.randn(N, Ho, Wo, Cout, device=DEV, generator=gen).bfloat16()
    return x, dy16


def _im2col_gemm(x, dy16, N, H, W, Cin, Cout, ldg, groups, stride, splits):
    """dW the way _conv_wgrad_tc computes it without the gathered path."""
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    Cig, Cog, M = Cin // groups, Cout // groups, N * Ho * Wo
    rows = max(Cout, ldg) if groups == 1 else Cout
    col = torch.empty((M, 9 * Cin), dtype=torch.bfloat16, device=DEV)
    _call('tfb_im2col3x3_bf16', x, col, N, H, W, Cin, stride, groups)
    dwp = torch.empty((rows, 9 * Cig), device=DEV)
    _call('tfb_gemm_bf16_tc_wgrad_batched', Cog if groups > 1 else rows, 9 * Cig, M, dy16, ldg, Cog if groups > 1 else 0, col, 9 * Cin,
          9 * Cig if groups > 1 else 0, dwp, 9 * Cig, Cog * 9 * Cig, groups, splits)
    return dwp[:Cout].reshape(Cout, Cig, 3, 3)


@pytest.mark.parametrize('cfg', CASES, ids=lambda c: 'N%d_%dx%d_%d-%d_ld%d_g%d_s%d_sp%d_cap%d' % c)
def test_conv3x3_wgrad_matches_im2col_gemm(cfg):
    N, H, W, Cin, Cout, ldg, groups, stride, splits, cap = cfg
    x, dy16 = _inputs(*cfg[:8])
    Cig = Cin // groups
    rows = max(Cout, ldg) if groups == 1 else Cout
    out = Guarded((Cout, Cig, 3, 3), torch.float32)
    work = torch.empty(rows * 9 * Cig, device=DEV)
    _call('tfb_gemm_set_max_ctas', cap)
    try:
        bits = []
        for _ in range(2):
            _call('tfb_conv3x3_tc_wgrad', x.bfloat16(), dy16, out.reset(), work, N, H, W, Cin, Cout, ldg, groups, stride, splits)
            torch.cuda.synchronize()
            assert out.tail_ok(), 'wrote past dW'
            bits.append(out.bits())
        ref = _im2col_gemm(x, dy16, N, H, W, Cin, Cout, ldg, groups, stride, splits)
        torch.cuda.synchronize()
    finally:
        _call('tfb_gemm_set_max_ctas', 0)
    assert torch.equal(bits[0], bits[1]), 'two runs differ'
    assert torch.equal(out.t.view(torch.int32), ref.contiguous().view(torch.int32)), 'differs from im2col + GEMM'
    w = torch.zeros(Cout, Cig, 3, 3, device=DEV)
    *_, r_dw, m_dw = R.conv3x3_ref(x, w, None, stride, groups, dy16[..., :Cout].float())
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    rel, ratio = R.check(out.t, r_dw, m_dw, N * Ho * Wo + 64, WGRAD_TOL, what='dw')
    print('wgrad %s: rel L2 %.2e, worst element %.4f of the bound' % (cfg, rel, ratio))


def test_conv3x3_wgrad_argument_checks():
    x, dy16 = _inputs(1, 8, 16, 64, 32, 32, 1, 1)
    x = x.bfloat16()
    dw = torch.full((32, 64, 3, 3), float('nan'), device=DEV)
    work = torch.empty(32 * 9 * 64, device=DEV)
    from transfuser_b200 import _lib
    bad = [
        (x, dy16, dw, work, 1, 8, 16, 60, 32, 32, 1, 1, 0),           # Cin not a multiple of 8
        (x, dy16, dw, work, 1, 8, 16, 64, 32, 30, 1, 1, 0),           # ldg not a multiple of 8
        (x, dy16, dw, work, 1, 8, 16, 64, 40, 32, 1, 1, 0),           # ldg < Cout
        (x, dy16, dw, work, 1, 8, 16, 64, 32, 32, 1, 3, 0),           # stride 3
        (x, dy16, dw, work, 1, 8, 16, 64, 36, 36, 3, 1, 0),           # 12-channel output groups
        (x[..., 1:], dy16, dw, work, 1, 8, 16, 64, 32, 32, 1, 1, 0),  # misaligned x
        (x, dy16, dw, None, 1, 8, 16, 64, 32, 32, 1, 1, 0),           # no work buffer
        (x, dy16, dw, work, 0, 8, 16, 64, 32, 32, 1, 1, 0),           # empty batch
    ]
    for a in bad:
        with pytest.raises(RuntimeError, match='failed with code'):
            _lib.call('tfb_conv3x3_tc_wgrad', *[t.data_ptr() if isinstance(t, torch.Tensor) else t for t in a])
    torch.cuda.synchronize()
    assert torch.isnan(dw).all(), 'a rejected call launched'


def _step(implicit, monkeypatch):
    import numpy as np
    import bench
    from transfuser_b200 import ops
    from transfuser_b200.config import TrainConfig
    from transfuser_b200.trainer import Trainer
    monkeypatch.setattr(ops, 'IMPLICIT_WGRAD', implicit)
    dev = torch.device(DEV, 0)
    host = bench.make_host_batch(2, seed=100, torch=torch, np=np, backbone='transFuser', raw=True)
    torch.manual_seed(0)                       # the initial weights
    tr = Trainer(TrainConfig(), dev, gemm_mode='bf16', lr=1e-4, seed=0, backbone='transFuser', raw_inputs=True)
    calls = []
    from transfuser_b200 import _lib
    L = _lib.lib()
    orig = L.call

    def spy(name, *a):
        calls.append(name)
        return orig(name, *a)

    L.call = spy
    try:
        tr.step({k: v.to(dev) for k, v in host.items()})
    finally:
        del L.call
    torch.cuda.synchronize()
    offs = dict(zip(map(id, tr.flat.params), tr.flat.offsets))
    grads = {n: tr.flat.grad[offs[id(p)]:offs[id(p)] + p.numel()].view(p.shape).clone() for n, p in tr.net.named_parameters()}
    return {k: v.clone() for k, v in tr.last_losses.items()}, grads, calls


def test_model_step_implicit_wgrad(monkeypatch):
    from transfuser_b200 import gemm
    old = gemm.MODE
    try:
        loss_a, grad_a, calls_a = _step(True, monkeypatch)
        loss_b, grad_b, calls_b = _step(False, monkeypatch)
    finally:
        gemm.set_mode(old)
    assert calls_a.count('tfb_conv3x3_tc_wgrad') >= 40 and 'tfb_im2col3x3_bf16' not in calls_a
    assert 'tfb_conv3x3_tc_wgrad' not in calls_b
    for k in loss_a:
        assert torch.equal(loss_a[k], loss_b[k]), k
    for n, a in grad_a.items():
        assert torch.equal(a.view(torch.int32), grad_b[n].view(torch.int32)), n
