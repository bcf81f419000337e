"""Throughput mode: bf16 operands on the wgmma tensor cores (fp32 accumulate, fp32 master weights / activations).
The per-op tests hold each product to the exact-operand reference of tests/tc_ref.py (the kernel's own bf16 operands contracted in
fp64: element-wise within the fp32 accumulation bound, relative L2 <= EXACT_TOL); against plain fp32 torch, bf16 keeps 8 mantissa
bits, so that secondary bound is 2e-2 relative L2 per op (the exact-fp32 mode is held to 1e-3 in test_ops.py / test_model.py)."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tc_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 2e-2
EXACT_TOL = 1e-4         # against the exact-operand references (fp32 accumulation order only)
# bf16 mode vs the oracle with bf16-rounded tensor-core operands: the errors grow from ~1e-3 at stage 1 to ~0.15 / 0.25 at stages
# 3 / 4 (against the fp32 oracle: ~7e-3 at stage 1 to ~0.24 / 0.38). Identical
# rounding POINTS do not give identical results at this test point: a 1e-7 difference in fp32 summation order flips a few bf16
# roundings per layer and the batch-2 network amplifies each flip ~100x by stage 4 (two runs of the SAME bf16 step differ by
# 0.4-1.5 % in the worst loss). The bounds are 3x the measured values for the early stages, loose beyond.
BF16_ORACLE_ACT_TOL = {'img_s1': 5e-3, 'lid_s1': 5e-3, 'img_s2': 4e-2, 'lid_s2': 4e-2}
BF16_ORACLE_LOSS_TOL = 0.2


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


def _spy(fn, keep=()):
    """(result, [(entry point, args)]) of the C-ABI calls fn() makes; for the entry points in `keep`, (args cloned before the call,
    args cloned after it), since the buffers may be reused later."""
    from transfuser_b200 import _lib
    L = _lib.lib()
    seen, orig = [], L.call

    def spy(name, *a):
        if name not in keep:
            seen.append((name, a))
            return orig(name, *a)
        clone = lambda args: [t.clone() if isinstance(t, torch.Tensor) else t for t in args]
        before = clone(a)
        r = orig(name, *a)
        seen.append((name, (before, clone(a))))
        return r

    L.call = spy
    try:
        out = fn()
    finally:
        del L.call
    return out, seen


def _names(calls):
    return [n for n, _ in calls]


def _exact_conv(x, w, b, stride, groups, dy, y, dx, dw, fwd_calls, bwd_calls):
    """A conv's output and gradients (NHWC x / y / dx / dy) against the exact-operand reference: bf16-rounded operands where the
    product ran on the tensor cores, the fp32 operands as given where it ran on a direct fp32 kernel (the narrow stems, small
    weight gradients)."""
    k = w.shape[2]
    Ho, Wo = y.shape[1], y.shape[2]
    refs = {}
    for rounding in (True, False):
        rx, rw, rg = (R.bf(x), R.bf(w), R.bf(dy)) if rounding else (x.double(), w.double(), dy.double())
        xn, gn = rx.permute(0, 3, 1, 2), rg.permute(0, 3, 1, 2)
        conv = lambda a, c: F.conv2d(a, c, None, stride=stride, padding=k // 2, groups=groups)
        ry, my = conv(xn, rw), conv(xn.abs(), rw.abs())
        if b is not None:
            ry, my = ry + b.double().view(1, -1, 1, 1), my + b.double().abs().view(1, -1, 1, 1)
        gin = lambda c, g: torch.nn.grad.conv2d_input(xn.shape, c, g, stride=stride, padding=k // 2, groups=groups)
        gw = lambda a, g: torch.nn.grad.conv2d_weight(a, rw.shape, g, stride=stride, padding=k // 2, groups=groups)
        refs[rounding] = [(ry, my), (gin(rw, gn), gin(rw.abs(), gn.abs())), (gw(xn, gn), gw(xn.abs(), gn.abs()))]
    fwd_tc = 'tfb_conv2d_fwd' not in _names(fwd_calls)
    dgrad_tc = 'tfb_conv2d_dgrad' not in _names(bwd_calls)
    wgrad_tc = 'tfb_conv2d_wgrad' not in _names(bwd_calls)
    kk = k * k * w.shape[1]
    res = []
    for i, (out, nhwc, rnd, K, what) in enumerate(((y, True, fwd_tc, kk + 2, 'y'), (dx, True, dgrad_tc, k * k * w.shape[0] // groups + 2, 'dx'),
                                                   (dw, False, wgrad_tc, dy.shape[0] * Ho * Wo + 64, 'dw'))):
        r, m = refs[rnd][i]
        if nhwc:
            r, m = r.permute(0, 2, 3, 1), m.permute(0, 2, 3, 1)
        res.append(R.check(out, r, m, K, EXACT_TOL, what=what + (' (bf16 operands)' if rnd else ' (fp32 operands)')))
    return res


@pytest.fixture(autouse=True)
def bf16_mode():
    from transfuser_b200 import gemm
    old = gemm.MODE
    gemm.set_mode('bf16')
    yield
    gemm.set_mode(old)


@pytest.mark.parametrize('M,K,N', [(348, 72, 72), (348, 216, 864), (1740, 1512, 1512), (14080, 72, 72), (70400, 32 + 40, 216), (200, 64, 64)])
def test_linear_bf16_fwd_bwd(M, K, N):
    from transfuser_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(M + K)
    x = torch.randn(M, K, device='cuda', generator=g).requires_grad_()
    w = (torch.randn(N, K, device='cuda', generator=g) / math.sqrt(K)).requires_grad_()
    b = torch.randn(N, device='cuda', generator=g).requires_grad_()
    xm, wm, bm = [t.detach().clone().requires_grad_() for t in (x, w, b)]
    yr = ops.linear(xm, wm, bm, relu=True)
    assert rel(yr, F.relu(F.linear(x, w, b))) < TOL   # fused bias + ReLU epilogue
    # exact operands: y = bf16(x) bf16(w)^T + b; dx = bf16(g) bf16(w); dw = bf16(g)^T bf16(x); db = sum g (fp32)
    ye, mag = R.contract(x.detach(), w.detach().t())
    R.check(yr, (ye + b.detach().double()).clamp_min(0), mag + b.detach().double().abs(), K + 2, EXACT_TOL, what='y (relu)')
    # gradients are compared without the ReLU: a bf16-perturbed pre-activation near 0 flips its mask, which is a property of
    # the comparison, not of the kernels
    ref = F.linear(x, w, b)
    out = ops.linear(xm, wm, bm, relu=False)
    assert rel(out, ref) < TOL
    R.check(out, ye + b.detach().double(), mag + b.detach().double().abs(), K + 2, EXACT_TOL, what='y')
    go = torch.randn(M, N, device='cuda', generator=g)
    mine = torch.autograd.grad(out, [xm, wm, bm], go)
    for a, r in zip(mine, torch.autograd.grad(ref, [x, w, b], go)):
        assert rel(a, r) < TOL
    R.check(mine[0], *R.contract(go, w.detach()), N + 2, EXACT_TOL, what='dx')
    R.check(mine[1], *R.contract(go.t(), x.detach()), M + 64, EXACT_TOL, what='dw')
    R.check(mine[2], go.double().sum(0), go.double().abs().sum(0), M + 2, EXACT_TOL, what='db')


def test_attention_bf16():
    from transfuser_b200 import ops
    B, T, C, nh = 2, 174, 216, 4
    g = torch.Generator(device='cuda').manual_seed(3)
    h = torch.randn(B * T, C, device='cuda', generator=g).requires_grad_()
    ws = [(torch.randn(C, C, device='cuda', generator=g) / math.sqrt(C)).requires_grad_() for _ in range(3)]
    bs = [(torch.randn(C, device='cuda', generator=g) * 0.1).requires_grad_() for _ in range(3)]
    q, k, v = [F.linear(h, ws[i], bs[i]).view(B, T, nh, C // nh).transpose(1, 2) for i in range(3)]
    ref = (F.softmax((q @ k.transpose(-2, -1)) / math.sqrt(C // nh), dim=-1) @ v).transpose(1, 2).reshape(B * T, C)
    hm = h.detach().clone().requires_grad_()
    wm = [w.detach().clone().requires_grad_() for w in ws]
    bm = [b.detach().clone().requires_grad_() for b in bs]
    go = torch.randn(B * T, C, device='cuda', generator=g)

    def run():
        out = ops.AttentionFn.apply(hm, wm[0], bm[0], wm[1], bm[1], wm[2], bm[2], B, T, nh, 0.0, 1)
        return out, torch.autograd.grad(out, [hm] + wm, go)
    (out, mine), calls = _spy(run, keep=('tfb_attn_fwd_tc',))
    assert rel(out, ref) < TOL
    for a, r in zip(mine, torch.autograd.grad(ref, [h] + ws, go)):
        assert rel(a, r) < 2 * TOL
    # the attention kernel's forward against the exact-operand reference of ITS q|k|v operand (the projection GEMM's bf16 output;
    # the kernel alone, backward included, is pinned in test_tc_exact.py)
    fwd = [a for n, a in calls if n == 'tfb_attn_fwd_tc']
    assert len(fwd) == 1
    before, after = fwd[0]
    qkv, Bk, Tk, nhk, hs = before[0].double(), before[2], before[3], before[4], before[5]
    assert (Bk, Tk, nhk, hs) == (B, T, nh, C // nh)
    y = after[6] if after[6] is not None else after[7]
    f = R.attn_fwd_ref(qkv, B, T, nh, hs, before[9], torch.ones(B, nh, T, T, dtype=torch.float64, device='cuda'))
    slack = f['y_slack'] + (0 if after[6] is not None else R.bf16_ulp(f['y'].abs() + f['y_K'] * R.EPS32 * f['y_mag'] + f['y_slack']))
    R.check(y, f['y'], f['y_mag'], f['y_K'], 1e-3 if after[6] is not None else 4e-3, slack, what='attention y')


@pytest.mark.parametrize('cfg', [
    # N, H, W, Cin, Cout, groups, bias, relu
    (2, 12, 20, 72, 72, 3, False, False),      # grouped, odd number of groups (last CTA holds one group)
    (1, 10, 44, 216, 216, 9, False, False),
    (2, 16, 16, 576, 576, 24, False, False),
    (1, 5, 22, 1512, 1512, 63, False, False),
    (2, 64, 64, 64, 64, 1, True, True),        # heads
    (1, 5, 22, 512, 128, 1, True, True),       # decoder: 8 K-chunks
    (2, 5, 22, 128, 64, 1, True, True),
    (1, 40, 176, 64, 32, 1, True, True),
    (1, 40, 48, 32, 32, 1, True, True),        # 32-channel rows (SWIZZLE_64B tiles)
    (2, 23, 37, 32, 7, 1, True, False),        # ragged tile edges, Cout 7
    (1, 16, 32, 32, 1, 1, True, False),
    (4, 40, 176, 32, 32, 1, True, False),      # long contraction: split-K wgrad
])
def test_conv3x3_tensor_core(cfg):
    from transfuser_b200 import ops
    N, H, W, Cin, Cout, g, has_b, relu = cfg
    gen = torch.Generator(device='cuda').manual_seed(Cin + Cout)
    x = torch.randn(N, Cin, H, W, device='cuda', generator=gen).requires_grad_()
    w = (torch.randn(Cout, Cin // g, 3, 3, device='cuda', generator=gen) / math.sqrt(Cin // g * 9)).requires_grad_()
    b = torch.randn(Cout, device='cuda', generator=gen).requires_grad_() if has_b else None
    ref = F.conv2d(x, w, b, padding=1, groups=g)
    xm = x.detach().permute(0, 2, 3, 1).contiguous().requires_grad_()
    wm = w.detach().clone().requires_grad_()
    bm = b.detach().clone().requires_grad_() if has_b else None
    assert ops._conv_tc_plan(Cin, Cout, g) is not None
    if relu:
        yr = ops.conv2d(xm, wm, bm, 1, g, True)
        assert rel(yr.permute(0, 3, 1, 2), F.relu(ref)) < TOL
    out, fwd_calls = _spy(lambda: ops.conv2d(xm, wm, bm, 1, g, False))
    assert rel(out.permute(0, 3, 1, 2), ref) < TOL
    go = torch.randn(N, Cout, H, W, device='cuda', generator=gen)
    gm = go.permute(0, 2, 3, 1).contiguous()
    mg, bwd_calls = _spy(lambda: torch.autograd.grad(out, [xm, wm], gm))
    rg = torch.autograd.grad(ref, [x, w], go)
    assert rel(mg[0].permute(0, 3, 1, 2), rg[0]) < TOL
    assert rel(mg[1], rg[1]) < TOL
    _exact_conv(xm.detach(), w.detach(), b.detach() if has_b else None, 1, g, gm, out.detach(), mg[0], mg[1], fwd_calls, bwd_calls)


def test_full_model_bf16_close_to_fp32_mode():
    """Throughput mode vs parity mode on the same weights / inputs: every loss within 5% of max(|loss|, 0.1)
    (bf16 operands, fp32 accumulate; the floor covers the near-zero yaw-residual SmoothL1 term)."""
    import sys
    import os
    sys.path.insert(0, os.path.dirname(__file__))
    from test_model import build
    from oracle import torch_oracle as O
    from transfuser_b200 import gemm
    batch = {k: v.cuda() for k, v in O.synthetic_batch(2, seed=3).items()}
    outs = {}
    for mode in ('simt', 'bf16'):
        gemm.set_mode(mode)
        net = build().cuda().train()
        out = net(batch['rgb'], batch['lidar'], ego_waypoint=batch['ego_waypoint'], target_point=batch['target_point'],
                  target_point_image=batch['target_point_image'], ego_vel=batch['ego_vel'], bev=batch['bev'], label=batch['label'],
                  depth=batch['depth'], semantic=batch['semantic'])
        outs[mode] = {k: v.item() for k, v in out.items()}
        sum(out.values()).backward()
        assert all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)
    for k in outs['simt']:
        a, b = outs['bf16'][k], outs['simt'][k]
        print('%-22s fp32 %.6f bf16 %.6f rel %.2e' % (k, b, a, abs(a - b) / max(abs(b), 1e-9)))
        # worst measured: loss_yaw_res 0.0142 vs 0.0172 (|diff| 3.0e-3) — a SmoothL1 over a handful of positive pixels that moves by
        # 5-20 % with any bf16 rounding flip upstream (smoke() bounds it at 35 %): absolute floor 0.2 * 5e-2 = 1e-2 for it
        assert abs(a - b) <= 5e-2 * max(abs(b), 0.2 if k == 'loss_yaw_res' else 0.1), (k, a, b)


@pytest.mark.parametrize('C', [72, 576, 1512])
def test_qkv_pack_fused_projection_bf16(C):
    """A GPT Block on flat parameters (optim.flatten packs query | key | value back to back): the fused [3C, C] projection (one
    tensor-core GEMM each for forward, dgrad, wgrad; one bias reduction) against the three-GEMM path on the same bf16 operands.
    Same products, different accumulation grouping: outputs and gradients agree to 1e-4 relative L2 (fp32 accumulation)."""
    from transfuser_b200 import gemm, ops, optim
    from transfuser_b200.backbone import Block
    B, T, nh = 10, 174, 4
    res = {}
    old = ops.QKV_FUSED
    try:
        for fused in (True, False):
            ops.QKV_FUSED = fused
            torch.manual_seed(3)
            blk = Block(C, nh, 4, 0.0, 0.0).cuda().train()
            fp = optim.flatten(blk)
            gemm.attach_bf16_weights(fp)
            a = blk.attn
            assert (ops._pack3(a.query.weight, a.key.weight, a.value.weight) is not None)
            x = torch.randn(B * T, C, device='cuda', generator=torch.Generator(device='cuda').manual_seed(4)).requires_grad_()
            y = blk.run(x, B, T)
            y.backward(torch.randn(B * T, C, device='cuda', generator=torch.Generator(device='cuda').manual_seed(5)))
            torch.cuda.synchronize()
            for p, o in zip(fp.params, fp.offsets):                  # gradients landed in the flat buffer, no copies
                assert p.grad is not None and p.grad.data_ptr() == fp.grad.data_ptr() + 4 * o
            res[fused] = [y.detach().clone(), x.grad.clone()] + [p.grad.clone() for _, p in sorted(blk.named_parameters())]
            names = ['y', 'dx'] + [n for n, _ in sorted(blk.named_parameters())]
    finally:
        ops.QKV_FUSED = old
    for n, u, v in zip(names, res[True], res[False]):
        if n == 'attn.key.bias':
            continue                                                 # true gradient 0 (softmax shift invariance): pure rounding noise
        assert rel(u, v) < 1e-4, (n, rel(u, v))


def test_bf16_sidecars_do_not_change_the_step():
    """bf16 sidecars (BatchNorm / SE / add / LayerNorm write the bf16 operand of the next GEMM in their own pass) against the
    separate cast launches they replace. The sidecar is the same rounding of the same fp32 value. Every reduction across CTAs
    is added in a fixed order, so two runs of the SAME configuration give the same bits (checked here); between the two
    configurations the launch structure differs, and one flipped bf16 rounding is amplified by the batch-2 BatchNorms, so the
    on/off difference is held to 1 % of the worst loss. The step needs > 100 fewer launches with the sidecars."""
    import sys
    import os
    sys.path.insert(0, os.path.dirname(__file__))
    from test_model import build
    from oracle import torch_oracle as O
    from transfuser_b200 import _lib, gemm, ops
    batch = {k: v.cuda() for k, v in O.synthetic_batch(2, seed=4).items()}
    gemm.set_mode('bf16')
    old = ops.SIDECARS

    def run(on):
        ops.SIDECARS = on
        net = build().cuda().train()
        n0 = _lib.lib().launches
        out = net(batch['rgb'], batch['lidar'], ego_waypoint=batch['ego_waypoint'], target_point=batch['target_point'],
                  target_point_image=batch['target_point_image'], ego_vel=batch['ego_vel'], bev=batch['bev'], label=batch['label'],
                  depth=batch['depth'], semantic=batch['semantic'])
        sum(out.values()).backward()
        torch.cuda.synchronize()
        assert all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)
        return {k: v.item() for k, v in out.items()}, _lib.lib().launches - n0

    def dist(a, b):
        return max(abs(a[k] - b[k]) / max(abs(b[k]), 0.1) for k in a)

    try:
        off0, l_off = run(False)
        off1, _ = run(False)
        off2, _ = run(False)
        on0, l_on = run(True)
        on1, _ = run(True)
    finally:
        ops.SIDECARS = old
    noise = max(dist(off0, off1), dist(off0, off2), dist(off1, off2), dist(on0, on1))
    worst = max(dist(on0, off0), dist(on1, off1), dist(on0, off2))
    print('bf16 step: run-to-run difference %.3e, sidecars on vs off %.3e; C-ABI calls %d -> %d' % (noise, worst, l_off, l_on))
    assert noise == 0.0, noise                      # repeat runs: the same bits
    assert worst <= 1e-2, worst
    assert l_off - l_on > 100


@pytest.mark.parametrize('cfg', [(2, 40, 48, 72, 72, 3), (2, 20, 24, 216, 216, 9), (2, 32, 44, 3, 32, 1)])
def test_conv3x3_stride2_bf16_mode(cfg):
    """Stride-2 3x3 convs (first block of every RegNetY stage, stems): forward on the tensor-core implicit-GEMM kernel whose TMA map
    steps two pixels per box element (the 3-channel stems stay on the exact fp32 direct kernel); dgrad as the stride-1
    tensor-core dgrad of the zero-dilated dy; wgrad through im2col + the batched tensor-core GEMM."""
    from transfuser_b200 import ops
    N, H, W, Cin, Cout, g = cfg
    gen = torch.Generator(device='cuda').manual_seed(Cin)
    x = torch.randn(N, Cin, H, W, device='cuda', generator=gen).requires_grad_()
    w = (torch.randn(Cout, Cin // g, 3, 3, device='cuda', generator=gen) / math.sqrt(Cin // g * 9)).requires_grad_()
    ref = F.conv2d(x, w, None, stride=2, padding=1, groups=g)
    xm = x.detach().permute(0, 2, 3, 1).contiguous().requires_grad_()
    wm = w.detach().clone().requires_grad_()
    out, fwd_calls = _spy(lambda: ops.conv2d(xm, wm, None, 2, g, False))
    assert rel(out.permute(0, 3, 1, 2), ref) < (TOL if (Cin % 8 == 0 and ops.CONV_S2_TC) else 1e-4)   # measured 2.4e-3 (bf16 operands)
    go = torch.randn_like(ref)
    gm = go.permute(0, 2, 3, 1).contiguous()
    mg, bwd_calls = _spy(lambda: torch.autograd.grad(out, [xm, wm], gm))
    rg = torch.autograd.grad(ref, [x, w], go)
    assert rel(mg[0].permute(0, 3, 1, 2), rg[0]) < TOL   # grouped: zero-dilated dy through the tensor-core dgrad
    assert rel(mg[1], rg[1]) < TOL
    _exact_conv(xm.detach(), w.detach(), None, 2, g, gm, out.detach(), mg[0], mg[1], fwd_calls, bwd_calls)


def test_conv1x1_stride2_bf16_mode():
    """RegNet downsample shortcut (1x1, stride 2): subsample + tensor-core GEMM; backward through the zero-dilation."""
    from transfuser_b200 import ops
    gen = torch.Generator(device='cuda').manual_seed(9)
    x = torch.randn(2, 72, 40, 48, device='cuda', generator=gen).requires_grad_()
    w = (torch.randn(216, 72, 1, 1, device='cuda', generator=gen) / math.sqrt(72)).requires_grad_()
    ref = F.conv2d(x, w, None, stride=2)
    xm = x.detach().permute(0, 2, 3, 1).contiguous().requires_grad_()
    wm = w.detach().clone().requires_grad_()
    out, fwd_calls = _spy(lambda: ops.conv2d(xm, wm, None, 2, 1, False))
    assert out.shape == (2, 20, 24, 216) and rel(out.permute(0, 3, 1, 2), ref) < TOL
    go = torch.randn_like(ref)
    gm = go.permute(0, 2, 3, 1).contiguous()
    mg, bwd_calls = _spy(lambda: torch.autograd.grad(out, [xm, wm], gm))
    rg = torch.autograd.grad(ref, [x, w], go)
    assert rel(mg[0].permute(0, 3, 1, 2), rg[0]) < TOL and rel(mg[1], rg[1]) < TOL
    _exact_conv(xm.detach(), w.detach(), None, 2, 1, gm, out.detach(), mg[0], mg[1], fwd_calls, bwd_calls)


@pytest.mark.parametrize('cfg', [(2, 20, 24, 72, 216, 1, 1, 1), (3, 10, 12, 216, 216, 3, 9, 1), (2, 20, 24, 72, 72, 3, 3, 2), (2, 9, 11, 576, 576, 1, 1, 1)])
def test_batchnorm_statistics_from_the_conv_epilogue(cfg):
    """conv (1x1 GEMM / grouped 3x3 / stride-2 3x3 on the tensor cores) + training-mode BatchNorm(+ReLU): the per-channel sum and
    sum of squares come out of the conv's epilogue (per-CTA partial sums, added in a fixed order into the per-step arena) and
    tfb_bn_fwd_stats normalises in one launch. Against torch conv + batch_norm on the bf16-rounded operands, and against the same product path with the fusion off."""
    from transfuser_b200 import _lib, ops
    N, H, W, Cin, Cout, k, g, stride = cfg
    gen = torch.Generator(device='cuda').manual_seed(Cin + Cout + k)
    x = torch.randn(N, Cin, H, W, device='cuda', generator=gen) * 1.5 + 0.3
    w = torch.randn(Cout, Cin // g, k, k, device='cuda', generator=gen) / math.sqrt(Cin // g * k * k)
    bn = torch.nn.BatchNorm2d(Cout).cuda().train()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5, generator=gen)
        bn.bias.uniform_(-0.3, 0.3, generator=gen)
    xr, wr = x.bfloat16().float(), w.bfloat16().float()
    yc = F.conv2d(xr, wr, None, stride=stride, padding=k // 2, groups=g)
    ref = F.relu(F.batch_norm(yc, None, None, bn.weight, bn.bias, True, 0.1, bn.eps))
    xm = x.permute(0, 2, 3, 1).contiguous()
    outs = {}
    old = ops.BN_STATS_FUSED
    try:
        for fused in (True, False):
            ops.BN_STATS_FUSED = fused
            bn.running_mean.zero_(); bn.running_var.fill_(1.0)
            ops.tick(x.device)
            y = ops.conv2d(xm, w, None, stride, g, False, bn_stats=True)
            assert (getattr(y, '_tfb_stats', None) is not None) == fused
            o = ops.batch_norm(y, bn, True, True)
            torch.cuda.synchronize()
            outs[fused] = (o.permute(0, 3, 1, 2).clone(), bn.running_mean.clone(), bn.running_var.clone())
    finally:
        ops.BN_STATS_FUSED = old
    assert rel(outs[True][0], ref) < 2e-3, rel(outs[True][0], ref)            # same bf16 operands, fp32 accumulation
    assert rel(outs[True][0], outs[False][0]) < 1e-5
    M = yc.numel() // Cout
    assert rel(outs[True][1], 0.1 * yc.mean((0, 2, 3))) < 1e-4
    assert rel(outs[True][2], 0.9 + 0.1 * yc.var((0, 2, 3), unbiased=True)) < 1e-4
    assert rel(outs[True][1], outs[False][1]) < 1e-5 and rel(outs[True][2], outs[False][2]) < 1e-5


def test_bf16_mode_matches_the_bf16_operand_oracle():
    """Parity in the mode bench.py times. The fp32 CPU oracle is the wrong yardstick for a bf16-operand run at this (batch 2,
    random weights) test point: ANY implementation that rounds the tensor-core operands to bf16 lands 24 % (stage 3) to 38 %
    (stage 4) away from the fp32 activations — the oracle itself does when told to round the same operands
    (oracle/torch_oracle.py BF16_OPERANDS: img_s3 0.240, img_s4 0.382 on the CPU; the CUDA path lands at the same distances).
    So the bf16 mode is held to the oracle evaluated WITH the product's rounding points
    (bf16 operands for every tensor-core contraction, fp32 accumulation, everything else fp32): per-stage activations and all 11
    losses, B = 2, dropout off."""
    import sys
    import os
    sys.path.insert(0, os.path.dirname(__file__))
    from test_model import build, rel as relm, _oracle_run
    from oracle import torch_oracle as O
    net0 = build()
    batch = O.synthetic_batch(2, seed=3)
    O.BF16_OPERANDS[0] = True
    try:
        P16, ref16, taps16 = _oracle_run(net0, batch, torch.float32)
    finally:
        O.BF16_OPERANDS[0] = False
    net = build().cuda().train()
    cb = {k: v.cuda() for k, v in batch.items()}
    mine = {}
    feats, grid, fused = net._model.forward_nhwc(cb['rgb'], torch.cat((cb['lidar'], cb['target_point_image']), dim=1), taps=mine)
    torch.cuda.synchronize()
    errs = {k: relm(mine[k].permute(0, 3, 1, 2), taps16[k]) for k in sorted(mine)}
    errs['p2'] = relm(feats[0].permute(0, 3, 1, 2), taps16['p2'])
    errs['img_grid'] = relm(grid.permute(0, 3, 1, 2), taps16['img_grid'])
    errs['fused'] = relm(fused, taps16['fused'])
    print('bf16 mode vs bf16-operand oracle:', {k: float('%.2e' % v) for k, v in errs.items()})
    net = build().cuda().train()
    out = net(cb['rgb'], cb['lidar'], ego_waypoint=cb['ego_waypoint'], target_point=cb['target_point'],
              target_point_image=cb['target_point_image'], ego_vel=cb['ego_vel'], bev=cb['bev'], label=cb['label'],
              depth=cb['depth'], semantic=cb['semantic'])
    lerr = {k: abs(out[k].item() - ref16[k].item()) / max(abs(ref16[k].item()), 1e-12) for k in ref16}
    print('losses:', {k: float('%.2e' % v) for k, v in lerr.items()})
    for k, v in errs.items():
        assert v < BF16_ORACLE_ACT_TOL.get(k, 0.6), (k, v)
    for k, v in lerr.items():
        assert v < BF16_ORACLE_LOSS_TOL, (k, v)
    # and the early stages sit closer to the bf16-operand oracle than to the fp32 one (6.6e-3 / 2.7e-2 measured against fp32)
    _, _, taps32 = _oracle_run(net0, batch, torch.float32)
    for k in ('img_s1', 'lid_s1', 'img_s2', 'lid_s2'):
        assert errs[k] < 0.7 * relm(mine[k].permute(0, 3, 1, 2), taps32[k]), k


@pytest.mark.parametrize('cfg', [(2, 40, 44, 72), (2, 24, 48, 216), (3, 10, 12, 576)])
def test_batchnorm_from_epilogue_statistics_with_se_pool(cfg):
    """The conv2.bn -> SE hand-off in bf16 mode: statistics from the conv epilogue, normalise + ReLU + the squeeze-excite average pool in
    ONE launch (the flat kernel for the narrow / tall maps, the slab kernel otherwise); pooled must equal the mean of the output."""
    from transfuser_b200 import ops
    N, H, W, C = cfg
    gen = torch.Generator(device='cuda').manual_seed(C + H)
    x = torch.randn(N, C, H, W, device='cuda', generator=gen) + 0.2
    w = torch.randn(C, C, 1, 1, device='cuda', generator=gen) / math.sqrt(C)
    bn = torch.nn.BatchNorm2d(C).cuda().train()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5, generator=gen)
        bn.bias.uniform_(-0.3, 0.3, generator=gen)
    yc = F.conv2d(x.bfloat16().float(), w.bfloat16().float())
    ref = F.relu(F.batch_norm(yc, None, None, bn.weight, bn.bias, True, 0.1, bn.eps))
    ops.tick(x.device)
    y = ops.conv2d(x.permute(0, 2, 3, 1).contiguous(), w, None, 1, 1, False, bn_stats=True)
    assert getattr(y, '_tfb_stats', None) is not None
    o = ops.batch_norm(y, bn, True, True, pool=True)
    torch.cuda.synchronize()
    assert rel(o.permute(0, 3, 1, 2), ref) < 2e-3
    pooled = getattr(o, '_tfb_pooled', None)
    assert pooled is not None and rel(pooled, ref.mean((2, 3))) < 2e-3
    assert rel(pooled, o.mean((1, 2))) < 1e-5
