"""The bf16 tensor-core kernels (fused attention, implicit-GEMM 3x3 conv, GEMM) against exact-operand references
(tests/tc_ref.py): the same bf16 operands contracted in fp64, compared element by element at the worst-case fp32 accumulation
bound. Outputs are pre-filled with NaN (every element must be written), and every case runs twice (the same bits).

The relative-L2 bounds are 10x the worst values measured on an H100 (noted next to each bound).
"""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tc_ref as R  # noqa: E402
from tc_ref import Guarded  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda'
# relative L2 against the rounding-point reference; measured worst 1.2e-4 (dk at hs 378, T 1, against the floored norm) and 1.0e-4
# (y at hs 378, T 129): 10x that is above the 1e-3 cap. Outputs written only in bf16 carry their own rounding (measured 1.7e-3 relative
# L2), so they are held to ATTN16_TOL; their element-wise check allows the allowance plus one bf16 ulp.
ATTN_TOL = 1e-3
ATTN16_TOL = 4e-3
CONV_TOL = 7e-5          # 10x the measured worst, 7.1e-6 (dw of the 1056-tile case)
PLAIN_TOL = 2e-2         # against the plain fp64 references (no rounding): a bound on bf16-operand error, not on the kernel
SEED = 0x5EED1234ABCD


def _call(name, *a):
    from transfuser_b200 import _lib
    _lib.call(name, *a)


# ------------------------------------------------------------------ attention
# every hs at T = 174 (the model's 18 / 54 / 144 / 378, plus sizes on the 64-column chunk and 128-column pass boundaries), and
# every T (around the 16-token k-steps, the 96-column backward halves, the 128-row tiles and the 192 limit) at hs = 18 and 378
HS = [18, 54, 144, 378, 2, 64, 128, 130]
TS = [1, 15, 16, 17, 96, 97, 127, 128, 129, 174, 191, 192]
ATTN_CASES = [(hs, 174) for hs in HS] + [(hs, T) for hs in (18, 378) for T in TS if T != 174]
OUTS = ['both', '32', '16']


def _attn_variant(i):
    """Case i's batch size, input dtype, outputs, y_bf16, p_drop and seed offset (cycled so that every combination is reached)."""
    outs = OUTS[i % 3]
    y_bf16 = 1 if outs == '16' else (0 if outs == '32' else (i // 3) % 2)
    return dict(B=(1, 3, 10)[i % 3 if i % 7 else 2], qkv_bf16=(i // 2) % 2, outs=outs, y_bf16=y_bf16,
                p=(0.0, 0.1, 0.5)[(i // 4) % 3 if i % 5 else 1], seed_off=(0, 7919)[(i // 3) % 2])


def _check_pair(t32, t16, ref, mag, K, slack, what, floor=0.0):
    """Checks the fp32 output (or, when only the bf16 one exists, the bf16 output with one more bf16 rounding allowed) and that the
    bf16 output is bf16(fp32 output) bit for bit."""
    res = []
    if t32 is not None:
        res.append(R.check(t32, ref, mag, K, ATTN_TOL, slack, what, floor))
        if t16 is not None:
            assert torch.equal(t16.view(torch.int16), t32.bfloat16().view(torch.int16)), '%s: bf16 output != bf16(fp32 output)' % what
    else:
        allow = K * R.EPS32 * mag + slack
        res.append(R.check(t16, ref, mag, K, ATTN16_TOL, slack + R.bf16_ulp(ref.abs() + allow), what + ' (bf16)', floor))
    return res[0]


@pytest.mark.parametrize('hs,T', ATTN_CASES)
def test_attention_exact(hs, T):
    i = ATTN_CASES.index((hs, T))
    v = _attn_variant(i)
    B, nh = v['B'], 4
    C, scale, p = nh * hs, R.scale_for(hs), v['p']
    g = torch.Generator(device=DEV).manual_seed(100 + i)
    qkv = torch.randn(B * T, 3 * C, device=DEV, generator=g)
    qkv[:, :C] *= 1.5                                                     # peakier softmax rows
    qkv_in = qkv.bfloat16() if v['qkv_bf16'] else qkv
    dy = torch.randn(B * T, C, device=DEV, generator=g)
    seed_dev = torch.tensor([SEED], dtype=torch.int64, device=DEV)
    want32, want16 = v['outs'] in ('both', '32'), v['outs'] in ('both', '16')
    y32 = Guarded((B * T, C), torch.float32) if want32 else None
    y16 = Guarded((B * T, C), torch.bfloat16) if want16 else None
    lse = Guarded((B, nh, T), torch.float32)
    d32 = Guarded((B * T, 3 * C), torch.float32) if want32 else None
    d16 = Guarded((B * T, 3 * C), torch.bfloat16) if want16 else None
    dsum = torch.empty((B, nh, T), device=DEV)
    dy16 = torch.empty((B * T, C), dtype=torch.bfloat16, device=DEV)
    outs = [o for o in (y32, y16, lse, d32, d16) if o is not None]
    runs = []
    for _ in range(2):
        for o in outs:
            o.reset()
        _call('tfb_attn_fwd_tc', qkv_in, v['qkv_bf16'], B, T, nh, hs, y32 and y32.t, y16 and y16.t, lse.t, scale, p, seed_dev,
              v['seed_off'])
        y_used = y16.t if v['y_bf16'] else y32.t
        _call('tfb_attn_bwd_tc', qkv_in, v['qkv_bf16'], dy, y_used, v['y_bf16'], lse.t, dsum, dy16, B, T, nh, hs, d32 and d32.t,
              d16 and d16.t, scale, p, seed_dev, v['seed_off'])
        torch.cuda.synchronize()
        assert all(o.tail_ok() for o in outs), 'write past the end of an output'
        runs.append([o.bits() for o in outs])
    assert all(torch.equal(a, b) for a, b in zip(*runs)), 'two launches differ'

    drop = R.drop_factor(SEED + v['seed_off'], B, nh, T, p, device=DEV)
    x = qkv_in.double()
    f = R.attn_fwd_ref(x, B, T, nh, hs, scale, drop)
    res = {'y': _check_pair(y32 and y32.t, y16 and y16.t, f['y'], f['y_mag'], f['y_K'], f['y_slack'], 'y')}
    res['lse'] = R.check(lse.t, f['lse'], torch.zeros_like(f['lse']), 0, ATTN_TOL, f['lse_slack'], 'lse')
    b = R.attn_bwd_ref(x, dy, y_used, lse.t, B, T, nh, hs, scale, drop)
    floor = 1e-2 * b['dqkv'].norm().item()          # dq / dk vanish for T = 1: relative L2 against the whole gradient's scale
    for j, name in enumerate(('dq', 'dk', 'dv')):
        sl = slice(j * C, (j + 1) * C)
        res[name] = _check_pair(d32 and d32.t[:, sl], d16 and d16.t[:, sl], b['dqkv'][:, sl], b['mag'][:, sl], b['K'], b['slack'][:, sl],
                                name, floor)
    # the plain fp64 attention (no rounding; the same mask): bounds the bf16-operand error, so the references cannot share a mistake
    yk = (y32.t if y32 is not None else y16.t)
    yp, _, _ = R.attn_plain(x, B, T, nh, hs, scale, drop)
    assert R.rel_l2(yk, yp.detach()) < PLAIN_TOL
    gp = R.attn_plain_grads(x, dy, B, T, nh, hs, scale, drop)
    dk = (d32.t if d32 is not None else d16.t).double()
    assert ((dk - gp).norm() / max(gp.norm().item(), 1e-30)).item() < PLAIN_TOL
    print('attention hs %d T %d %s: %s' % (hs, T, v, {k: '%.2e / %.4f' % r for k, r in res.items()}))


def test_attention_argument_checks():
    """Shapes the kernel cannot serve are refused on the host, before any launch."""
    seed_dev = torch.zeros(1, dtype=torch.int64, device=DEV)
    qkv = torch.zeros(2 * 193 * 3 * 4 * 18 + 8, device=DEV)
    y, lse = torch.empty(2 * 193 * 72 + 8, device=DEV), torch.empty(2 * 4 * 193, device=DEV)
    for args in [(qkv, 0, 2, 193, 4, 18),                    # T > 192
                 (qkv, 0, 2, 50, 4, 17),                     # odd head size
                 (qkv[2:], 0, 2, 50, 4, 18)]:                # qkv not 16-byte aligned
        with pytest.raises(RuntimeError, match='argument check failed'):
            _call('tfb_attn_fwd_tc', *args, y, None, lse, 0.2, 0.0, seed_dev, 0)
        with pytest.raises(RuntimeError, match='argument check failed'):
            _call('tfb_attn_bwd_tc', args[0], 0, y, y, 0, lse, lse, y, *args[2:], y, None, 0.2, 0.0, seed_dev, 0)


# ------------------------------------------------------------------ 3x3 convolution
def _spy(fn):
    """(result, [(entry point, args)]) of the C-ABI calls fn() makes."""
    from transfuser_b200 import _lib
    L = _lib.lib()
    seen, orig = [], L.call

    def spy(name, *a):
        seen.append((name, a))
        return orig(name, *a)

    L.call = spy
    try:
        out = fn()
    finally:
        del L.call
    return out, seen


def _plans(calls):
    return [(a[10], a[9]) for n, a in calls if n in ('tfb_conv3x3_tc', 'tfb_conv3x3_tc_strided')]      # (KC, NB)


CONV_CASES = [
    # N, H, W, Cin, Cout, groups, stride, bias, relu, forward (KC, NB), dgrad (KC, NB); >= 512 output pixels (wgrad on the tensor cores)
    (2, 23, 37, 40, 16, 1, 1, True, False, (64, 16), (32, 64)),       # Cin 40: a partial 64-channel chunk
    (2, 17, 20, 16, 40, 1, 1, False, False, (32, 64), (64, 16)),
    (3, 9, 30, 8, 24, 1, 1, True, True, (32, 32), (32, 16)),
    (2, 16, 18, 32, 16, 1, 1, False, True, (32, 16), (32, 32)),
    (2, 14, 19, 32, 48, 1, 1, False, False, (32, 64), (64, 32)),
    (2, 14, 20, 136, 136, 1, 1, True, False, (64, 128), (64, 128)),   # 136 = 2 * 64 + 8; two output-channel blocks
    (2, 16, 16, 64, 64, 1, 1, False, False, (64, 64), (64, 64)),
    (2, 14, 20, 72, 72, 3, 1, False, False, (64, 48), (64, 48)),      # grouped, odd group count
    (3, 23, 37, 64, 32, 1, 2, True, False, (64, 32), (32, 64)),       # stride 2, odd sizes
    (4, 24, 26, 216, 216, 9, 2, False, False, (64, 48), (64, 48)),    # stride 2 grouped
    (8, 96, 176, 64, 128, 1, 1, False, False, (64, 128), (64, 64)),   # 1056 tiles: ~8 per persistent CTA
]


@pytest.fixture
def bf16_mode():
    from transfuser_b200 import gemm
    old = gemm.MODE
    gemm.set_mode('bf16')
    yield
    gemm.set_mode(old)


@pytest.mark.parametrize('cfg', CONV_CASES, ids=lambda c: 'N%d_%dx%d_%d-%d_g%d_s%d' % c[:7])
def test_conv3x3_exact(cfg, bf16_mode):
    from transfuser_b200 import ops
    N, H, W, Cin, Cout, groups, stride, has_b, relu, pf, pd = cfg
    gen = torch.Generator(device=DEV).manual_seed(Cin * 7 + Cout + H)
    x = torch.randn(N, H, W, Cin, device=DEV, generator=gen)
    w = torch.randn(Cout, Cin // groups, 3, 3, device=DEV, generator=gen) / math.sqrt(Cin // groups * 9)
    bias = torch.randn(Cout, device=DEV, generator=gen) if has_b else None
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    dy = torch.randn(N, Ho, Wo, Cout, device=DEV, generator=gen)

    def run():
        xm, wm = x.clone().requires_grad_(), w.clone().requires_grad_()
        bm = bias.clone().requires_grad_() if has_b else None
        y = ops.conv2d(xm, wm, bm, stride, groups, relu)
        dx, dw = torch.autograd.grad(y, [xm, wm], dy)
        torch.cuda.synchronize()
        return y.detach(), dx, dw

    runs = [_spy(run) for _ in range(2)]
    (y, dx, dw), calls = runs[0]
    for a, b in zip(runs[0][0], runs[1][0]):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), 'two runs differ'
    plans = _plans(calls)
    assert plans == [pf, pd], plans
    assert 'tfb_gemm_bf16_tc_wgrad_batched' in [n for n, _ in calls]
    mask = (y > 0).float() if relu else 1.0
    r_y, m_y, r_dx, m_dx, r_dw, m_dw = R.conv3x3_ref(x, w, bias, stride, groups, dy * mask)
    if relu:
        r_y = r_y.clamp_min(0)
    K = 9 * Cin // groups
    res = [R.check(y, r_y, m_y, K + 2, CONV_TOL, what='y')]
    res.append(R.check(dx, r_dx, m_dx, 9 * Cout // groups + 2, CONV_TOL, what='dx'))
    res.append(R.check(dw, r_dw, m_dw, N * Ho * Wo + 64, CONV_TOL, what='dw'))
    # and against the plain fp32-operand conv (no rounding) at the bf16-operand bound
    import torch.nn.functional as F
    yp = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), bias.double() if has_b else None, stride=stride, padding=1, groups=groups)
    assert R.rel_l2(y.permute(0, 3, 1, 2), yp.clamp_min(0) if relu else yp) < PLAIN_TOL
    print('conv %s: plans fwd %s dgrad %s; y/dx/dw %s' % (cfg[:9], pf, pd, ['%.2e / %.4f' % r for r in res]))


@pytest.mark.parametrize('cfg', [(2, 20, 24, 72, 216, 1, 1, 1, 0.0), (2, 20, 24, 72, 72, 3, 3, 1, 0.0), (2, 21, 26, 64, 64, 3, 1, 2, 0.0),
                                 (4, 40, 44, 64, 64, 3, 1, 1, 0.62)], ids=['1x1', 'grouped', 'stride2', 'mean10std'])
def test_conv_epilogue_statistics(cfg, bf16_mode):
    """The BatchNorm statistics of the conv / GEMM epilogue: sum and sum of squares against fp64 sums of the kernel's own fp32
    output, and the variance derived from them (what BatchNorm uses) against a two-pass fp64 variance. The last case has a
    channel mean about 10x its standard deviation, where E[y^2] - E[y]^2 cancels two digits."""
    from transfuser_b200 import ops
    N, H, W, Cin, Cout, k, groups, stride, shift = cfg
    gen = torch.Generator(device=DEV).manual_seed(Cin + Cout + H)
    x = torch.randn(N, H, W, Cin, device=DEV, generator=gen) + shift
    w = torch.randn(Cout, Cin // groups, k, k, device=DEV, generator=gen) / math.sqrt(Cin // groups * k * k)
    if shift:       # mean ~ shift, std ~ 1 / sqrt(9 Cin) = 1 / 24: |mean| / std ~ 24 shift
        w = (1 + 0.1 * w * math.sqrt(Cin * k * k)) / (Cin * k * k)
    sums = []
    for _ in range(2):
        ops.tick(x.device)
        y = ops.conv2d(x, w, None, stride, groups, False, bn_stats=True)
        st = getattr(y, '_tfb_stats', None)
        assert st is not None
        torch.cuda.synchronize()
        sums.append((y.clone(), st.clone()))
    assert torch.equal(sums[0][0], sums[1][0]) and torch.equal(sums[0][1], sums[1][1]), 'two runs differ'
    y, st = sums[0]
    yd = y.double().reshape(-1, Cout)
    M = yd.shape[0]
    R.check(st[:Cout], yd.sum(0), yd.abs().sum(0), M + 16, 1e-4, what='sum')
    R.check(st[Cout:], (yd * yd).sum(0), (yd * yd).sum(0), M + 16, 1e-4, what='sum of squares')
    mean = st[:Cout] / M
    var = st[Cout:] / M - mean * mean
    var_ref = yd.var(0, unbiased=False)
    ratio = (yd.mean(0).abs() / var_ref.sqrt()).max().item()
    err = ((var - var_ref).abs() / var_ref).max().item()
    print('statistics %s: |mean| / std up to %.1f, variance from the epilogue sums: worst relative error %.2e' % (cfg, ratio, err))
    if shift:
        assert ratio > 8
    assert err < 1e-4, err


# ------------------------------------------------------------------ GEMM (one subprocess per forced tile width)
@pytest.mark.parametrize('width', [32, 64, 96, 128, 160, 192])
def test_gemm_bf16_exact(width):
    """Every K-major tile width (32 ... 192; MN-major B rounds the forced width up to 64 / 128 / 192): all four layouts, M across the
    128-row tiles, N ragged, K from 16 to 6048, alpha / bias / ReLU / beta, split-K (explicit and automatic), the scalar epilogue,
    the grid cap (bitwise), the bf16 output (bitwise = bf16(fp32)), the statistics epilogue and the batched weight gradient."""
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'tc_gemm_worker.py')
    env = dict(os.environ, TFB_GEMM_BN=str(width))
    cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [worker, str(width)]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out['width'] == width
    bad = [c for c in out['cases'] if c['error']]
    for c in out['cases']:
        print('gemm width %d %-34s %s' % (width, c['case'], c['error'] or 'rel %.2e ratio %.4f' % (c['rel'], c['ratio'])))
    assert not bad, '\n'.join('%s: %s\n%s' % (c['case'], c['error'], c.get('tb', '')) for c in bad)
    assert len(out['cases']) >= 30
