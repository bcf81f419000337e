"""The loss kernels of csrc/losses.cu (cross-entropy, L1, tfb_ratio, the CenterNet targets and the seven CenterNet head losses),
forward and backward, against float64 evaluations of the reference's formulas on the same fp32 inputs.

Tolerances follow from the arithmetic, not from the errors seen in a run:
  - forward totals: relative error <= max(2e-6, 4 x the relative error of torch evaluating the same formula in fp32);
  - gradients, element by element: every element is coef * w_m * (a term of magnitude <= 1), so |d - d64| <= 1e-6 * |coef * w_m|.
    The focal term of the heatmap has log(1 - sigmoid(x)) in it, and fp32's 1 - sigmoid(x) is off by up to 2^-25 absolutely, so its
    bound is 1e-6 * |coef| * (2 + |x|).
Heatmap logits are kept to |x| <= 12 except in the saturation test: beyond ~16 the eps-regularised logs of the focal loss legitimately
differ between fp32 and fp64, and the reference itself runs in fp32, so there the fp32 evaluation of the oracle is the reference."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import torch_oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda'   # tests/test_losses_emulated.py re-runs these functions with DEV = 'cpu' over the CPU emulation of the kernels
# rows: one; one block less a thread; two blocks; the CenterNet map at batch 10 (10*64*64); the semantic map at batch 10 (10*160*704)
CE_M = (1, 255, 257, 40960, 1126400)
L1_N = (1, 3, 1027, 1126400)            # the last: the depth map at batch 10
REGIME_M = 4096
CE_IDS = ('one-row', 'one-block', 'two-blocks', 'centernet-map', 'semantic-map')

RATIO = 64 / 256                          # 64x64 head map over the 256-px BEV
HEAD = (('loss_center_heatmap', 0, 1), ('loss_wh', 1, 3), ('loss_offset', 3, 5), ('loss_yaw_class', 5, 17), ('loss_yaw_res', 17, 18),
        ('loss_velocity', 18, 19), ('loss_brake', 19, 21))      # loss name, columns of pred[..., 21]
LW, DIV = (1.0, 0.1, 1.0, 1.0, 1.0, 1.0, 1.0), (1, 2, 2, 1, 1, 1, 1)
GOUT = (1.0, 0.3, 0.7, 1.3, 0.9, 1.7, 0.4)                        # seven distinct upstream gradients: a swapped coefficient shows


def _call(name, *args):
    from transfuser_b200._lib import call
    call(name, *args)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _bits(t):
    return t.detach().cpu().view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def _twice(name, args, acc):
    """Runs a forward entry point twice: its fp64 accumulators must come out with the same bits."""
    _call(name, *args)
    first = acc.clone()
    _call(name, *args)
    assert torch.equal(_bits(first), _bits(acc)), (name, first, acc)


def _check_total(got, ref64, ref32, what):
    """A forward total: relative error <= max(2e-6, 4 x torch fp32's relative error on the same inputs); exactly 0 where the
    float64 value is 0."""
    got, ref64, ref32 = (float(v.detach()) if torch.is_tensor(v) else float(v) for v in (got, ref64, ref32))
    if ref64 == 0.0:
        assert got == 0.0, (what, got)
        return
    err, terr = abs(got - ref64) / abs(ref64), abs(ref32 - ref64) / abs(ref64)
    assert err <= max(2e-6, 4 * terr), (what, got, ref64, err, terr)


def _check_grad(d, d64, bound, what):
    """Element by element: d finite and |d - d64| <= bound (an exact 0 where the bound is 0)."""
    d, d64, bound = d.detach().double().cpu(), d64.detach().double().cpu(), bound.double().cpu().expand_as(d64)
    assert torch.isfinite(d).all(), what
    excess = (d - d64).abs() - bound
    if (excess > 0).any():
        i = int(excess.flatten().argmax())
        raise AssertionError('%s: %d elements outside the bound; worst: got %r, float64 %r, bound %r'
                             % (what, int((excess > 0).sum()), d.flatten()[i].item(), d64.flatten()[i].item(), bound.flatten()[i].item()))


# ------------------------------------------------------------------ cross-entropy
def _ce_ref(x, t, class_w=None, pos_w=None, HW=1):
    """float64 on the fp32 logits: the leaf, nll_m and w_m = class_w[t_m] * pos_w[m % HW] (include/tfb200.h)."""
    x64 = x.double().requires_grad_()
    nll = -torch.log_softmax(x64, 1).gather(1, t[:, None])[:, 0]
    w = torch.ones(x.shape[0], dtype=torch.float64, device=x.device)
    if class_w is not None:
        w = w * class_w.double()[t]
    if pos_w is not None:
        w = w * pos_w.double()[torch.arange(x.shape[0], device=x.device) % HW]
    return x64, nll, w


def _ce_fwd(x, t, class_w=None, pos_w=None, HW=1):
    M, C = x.shape
    acc = torch.empty(2, dtype=torch.float64, device=DEV)
    _twice('tfb_ce_fwd', (x, t, M, C, class_w, pos_w, HW, acc), acc)
    return acc


def _check_ce_op(x, t, class_w, x64, nll, w, k=1.7, g=0.7):
    """ops.CrossEntropyFn in both denominator modes: the loss against float64, and every logit's gradient against float64 autograd
    within 1e-6 * |coef * w_m|, coef = g * k / den."""
    from transfuser_b200 import ops
    M = x.shape[0]
    w32 = class_w[t] if class_w is not None else torch.ones(M, device=DEV)
    for den_mode in ('wsum', 'count'):
        xm = x.clone().requires_grad_()
        out = ops.CrossEntropyFn.apply(xm, t, class_w, den_mode, k)
        den = w.sum() if den_mode == 'wsum' else float(M)
        ref = k * (w * nll).sum() / den
        ref32 = k * (F.cross_entropy(x, t, reduction='none') * w32).sum() / (w32.sum() if den_mode == 'wsum' else M)
        _check_total(out, ref, ref32, ('loss', den_mode))
        (d,) = torch.autograd.grad(out, xm, torch.tensor(g, device=DEV))
        (d64,) = torch.autograd.grad(ref * g, x64, retain_graph=True)
        _check_grad(d, d64, 1e-6 * (g * k / den * w).abs()[:, None], ('dlogits', den_mode))


@pytest.mark.parametrize('weighted', [False, True])
@pytest.mark.parametrize('mi', range(5), ids=CE_IDS)
@pytest.mark.parametrize('C', [2, 3, 7, 12, 16])
def test_cross_entropy_sizes(C, mi, weighted):
    """Grid-stride loops and the multi-block fold at every row count, class counts up to kMaxC = 16, with and without class weights."""
    M = CE_M[mi]
    g = _gen(100 * C + mi)
    x = (torch.randn(M, C, generator=g) * 3).to(DEV)
    t = torch.randint(0, C, (M,), generator=g).to(DEV)
    cw = (torch.rand(C, generator=g) * 2 + 0.25).to(DEV) if weighted else None
    acc = _ce_fwd(x, t, cw)
    x64, nll, w = _ce_ref(x, t, cw)
    w32 = cw[t] if weighted else torch.ones(M, device=DEV)
    _check_total(acc[0], (w * nll).sum(), (F.cross_entropy(x, t, reduction='none') * w32).sum(), 'sum w*nll')
    _check_total(acc[1], w.sum(), w32.sum(), 'sum w')
    _check_ce_op(x, t, cw, x64, nll, w)


def _regime_logits(regime, M, C, t, g):
    if regime == 'random':
        return torch.randn(M, C, generator=g) * 3
    if regime in ('confident', 'shifted'):                  # the right class ahead by 9: row losses ~1e-3
        x = torch.randn(M, C, generator=g)
        x[torch.arange(M), t] += 9.0
        return x + 1000.0 if regime == 'shifted' else x     # shifted: the softmax is the same, the logits are large
    if regime == 'saturated':
        return torch.where(torch.rand(M, C, generator=g) < 0.5, 80.0, -80.0)
    return (torch.randn(M, 1, generator=g) * 3).expand(M, C).contiguous()   # 'equal': every row's loss is log C


@pytest.mark.parametrize('regime', ['random', 'confident', 'shifted', 'saturated', 'equal'])
@pytest.mark.parametrize('C', [2, 7, 16])
def test_cross_entropy_logit_regimes(C, regime):
    """Confident and shifted logits: the row loss must be formed as log(se) - (x_t - max), the way torch's log_softmax does;
    adding the max first loses the low bits of log(se)."""
    M = REGIME_M
    g = _gen(7 * C + len(regime))
    t = torch.randint(0, C, (M,), generator=g)
    x = _regime_logits(regime, M, C, t, g).to(DEV)
    t = t.to(DEV)
    cw = (torch.rand(C, generator=g) + 0.5).to(DEV)
    acc = _ce_fwd(x, t, cw)
    x64, nll, w = _ce_ref(x, t, cw)
    _check_total(acc[0], (w * nll).sum(), (F.cross_entropy(x, t, reduction='none') * cw[t]).sum(), ('sum w*nll', regime))
    if regime == 'equal':
        assert abs(float(acc[0]) / float(w.sum()) - math.log(C)) <= 2e-6 * math.log(C)
    _check_ce_op(x, t, cw, x64, nll, w)


@pytest.mark.parametrize('weighted', [False, True])
@pytest.mark.parametrize('B,HW', [(3, 77), (10, 4096)])
def test_cross_entropy_position_weights(B, HW, weighted):
    """The pos_w argument of tfb_ce_fwd / tfb_ce_bwd: a per-position weight broadcast over the batch, w_m = class_w[t_m] * pos_w[m % HW],
    with both denominators (the weight sum from the forward accumulator, and none)."""
    M, C = B * HW, 7
    g = _gen(B + HW + weighted)
    x = (torch.randn(M, C, generator=g) * 3).to(DEV)
    t = torch.randint(0, C, (M,), generator=g).to(DEV)
    pw = torch.rand(HW, generator=g) * 2
    pw[::13] = 0.0
    pw = pw.to(DEV)
    cw = (torch.rand(C, generator=g) * 2 + 0.25).to(DEV) if weighted else None
    acc = _ce_fwd(x, t, cw, pw, HW)
    x64, nll, w = _ce_ref(x, t, cw, pw, HW)
    w32 = (cw[t] if weighted else torch.ones(M, device=DEV)) * pw[torch.arange(M, device=DEV) % HW]
    _check_total(acc[0], (w * nll).sum(), (F.cross_entropy(x, t, reduction='none') * w32).sum(), 'sum w*nll')
    _check_total(acc[1], w.sum(), w32.sum(), 'sum w')
    gout = torch.tensor([0.7], device=DEV)
    for den, k in ((acc[1:], 1.3), (None, 1.0 / M)):
        d = torch.empty_like(x)
        _call('tfb_ce_bwd', x, t, M, C, cw, pw, HW, gout, den, 0.0, k, d)
        den64 = w.sum() if den is not None else 1.0
        (d64,) = torch.autograd.grad(0.7 * k * (w * nll).sum() / den64, x64, retain_graph=True)
        _check_grad(d, d64, 1e-6 * (0.7 * k / den64 * w).abs()[:, None], ('dlogits', den is not None))


def test_cross_entropy_zero_weights_and_ratio_clamp():
    """All-zero weights give a zero weight sum: den_min keeps the loss and the gradient at 0 instead of 0/0. tfb_ratio itself:
    out = fp32(k * num / max(den, den_min)) in double, or k * num without a denominator."""
    M, C = 300, 5
    g = _gen(5)
    x = (torch.randn(M, C, generator=g) * 3).to(DEV)
    t = torch.randint(0, C, (M,), generator=g).to(DEV)
    cw = torch.zeros(C, device=DEV)
    acc = _ce_fwd(x, t, cw)
    assert acc.tolist() == [0.0, 0.0]
    out = torch.empty((), device=DEV)
    _call('tfb_ratio', acc, acc[1:], 1e-6, 1.0, out)
    assert out.item() == 0.0
    d = torch.full_like(x, float('nan'))
    _call('tfb_ce_bwd', x, t, M, C, cw, None, 1, torch.tensor([0.7], device=DEV), acc[1:], 1e-6, 1.0, d)
    assert torch.equal(d, torch.zeros_like(d))
    num = 3.7
    for den in (None, 0.25, 1e-9):
        for den_min, k in ((0.0, 1.0), (1e-6, 0.3), (0.5, 1.7)):
            nd = torch.tensor([num], dtype=torch.float64, device=DEV)
            dd = torch.tensor([den], dtype=torch.float64, device=DEV) if den is not None else None
            _call('tfb_ratio', nd, dd, den_min, k, out)
            want = np.float64(np.float32(k)) * num
            if den is not None:
                want /= max(den, np.float64(np.float32(den_min)))
            assert out.item() == float(np.float32(want)), (den, den_min, k, out.item(), want)


def test_loss_entry_points_refuse_bad_shapes():
    """More than kMaxC = 16 classes, or no rows, is an error, not a silent wrong answer."""
    from transfuser_b200 import ops
    x, t = torch.randn(8, 17, device=DEV), torch.randint(0, 17, (8,), device=DEV)
    with pytest.raises(RuntimeError):
        ops.CrossEntropyFn.apply(x, t, None, 'count', 1.0)
    with pytest.raises(RuntimeError):
        _call('tfb_ce_bwd', x, t, 8, 17, None, None, 1, None, None, 0.0, 1.0, torch.empty_like(x))
    with pytest.raises(RuntimeError):
        ops.CrossEntropyFn.apply(torch.empty(0, 7, device=DEV), torch.empty(0, dtype=torch.int64, device=DEV), None, 'count', 1.0)
    with pytest.raises(RuntimeError):
        _call('tfb_l1_fwd', x, x, 0, 0, torch.empty(1, dtype=torch.float64, device=DEV))


# ------------------------------------------------------------------ L1
@pytest.mark.parametrize('ni', range(4), ids=('one', 'three', 'odd', 'depth-map'))
@pytest.mark.parametrize('sigmoid', [False, True])
def test_l1(sigmoid, ni):
    """k * mean |f(x) - t|, f = sigmoid or identity. Every fifth element (from the second) is a tie, d == 0, whose gradient is 0 as in
    torch; with the sigmoid, another fifth is saturated at +-30, and the ties sit at x = 30, t = 1 (sigmoid rounds to 1 in fp32)."""
    from transfuser_b200 import ops
    n, k, gscale = L1_N[ni], 10.0, 0.7
    g = _gen(11 * ni + sigmoid)
    x = torch.randn(n, generator=g) * 2
    i = torch.arange(n)
    tie = i % 5 == 1
    if sigmoid:
        t = torch.rand(n, generator=g)
        sat = i % 5 == 3
        x[sat] = torch.where(i[sat] % 2 == 0, 30.0, -30.0)
        x[tie], t[tie] = 30.0, 1.0
        # the residual's sign must not hang on the rounding of sigmoid: keep the others at least 1e-5 from it
        near = ((x.double().sigmoid() - t.double()).abs() < 1e-5) & ~tie
        t[near] = t[near] + 3e-5
    else:
        t = torch.randn(n, generator=g)
        t[tie] = x[tie]
    x, t, tie = x.to(DEV), t.to(DEV), tie.to(DEV)
    f32 = torch.sigmoid(x) if sigmoid else x
    acc = torch.empty(1, dtype=torch.float64, device=DEV)
    _twice('tfb_l1_fwd', (x, t, n, int(sigmoid), acc), acc)
    x64 = x.double().requires_grad_()
    r = ((x64.sigmoid() if sigmoid else x64) - t.double()).abs()
    _check_total(acc[0], r.sum(), (f32 - t).abs().sum(), 'sum |d|')
    xm = x.clone().requires_grad_()
    out = ops.L1Fn.apply(xm, t, sigmoid, k)
    ref = k * r.sum() / n
    _check_total(out, ref, k * F.l1_loss(f32, t), 'loss')
    (d,) = torch.autograd.grad(out, xm, torch.tensor(gscale, device=DEV))
    (d64,) = torch.autograd.grad(ref * gscale, x64)
    _check_grad(d, d64, torch.full((1,), 1e-6 * gscale * k / n), 'dx')
    xt = x.clone().requires_grad_()
    (dt,) = torch.autograd.grad(F.l1_loss(torch.sigmoid(xt) if sigmoid else xt, t, reduction='sum'), xt)
    assert (d[tie] == 0).all() and (dt[tie] == 0).all()


# ------------------------------------------------------------------ CenterNet
def _random_boxes(n, g):
    r = lambda *s: torch.rand(*s, generator=g)
    b = torch.zeros(n, 7)
    b[:, 0:2] = r(n, 2) * 253 + 1
    b[:, 2:4] = r(n, 2) * 32 + 8
    b[:, 4] = r(n) * 2 * np.pi - np.pi
    b[:, 5] = r(n) * 8
    b[:, 6] = (r(n) < 0.5).float()
    return b


BORDER = torch.tensor([[0.2, 0.3, 60., 30., 0.0, 1., 0.], [255.9, 0.1, 8., 8., np.pi, 2., 1.], [0.4, 255.8, 100., 4., -np.pi, 0., 1.],
                       [255.7, 255.9, 2., 2., 2 * np.pi / 12, 3., 0.], [128.0, 0.0, 16., 90., -np.pi / 12, 1., 1.],
                       [3.99, 251.9, 33., 12., 7.5, 4., 0.]])


def _labels(kind, B, seed):
    """[B, 20, 7] label sets. 'border': centres in the first / last cells, in every sample (so every occupied cell is occupied in
    all B samples); 'coincident': two boxes in one cell; 'shared': three cells occupied in every sample next to boxes of its own."""
    g = _gen(seed)
    label = torch.zeros(B, 20, 7)
    common = _random_boxes(3, g)
    for b in range(B):
        if kind == 'random':
            label[b] = _random_boxes(20, g)
        elif kind == 'border':
            label[b, :3], label[b, 4:7] = BORDER[:3], BORDER[3:]     # row 3: a gap
        elif kind == 'coincident':
            label[b, :6] = _random_boxes(6, g)
            label[b, 6] = _random_boxes(1, g)[0]
            label[b, 6, 0:2] = torch.floor(label[b, 0, 0:2] / 4) * 4 + torch.tensor([3.7, 0.2])   # the same 4-px cell as box 0
        elif kind == 'shared':
            label[b, :3] = common
            label[b, 3:10] = _random_boxes(7, g)
    return label


def _edge_labels():
    """Five samples: none; 20 random boxes; the border boxes; two boxes in one cell and a gap row; one box after zero rows. Yaw angles
    on bin boundaries and outside [-pi, pi]."""
    g = _gen(9)
    label = torch.zeros(5, 20, 7)
    label[1] = _random_boxes(20, g)
    label[2, :6] = BORDER
    label[3, 0] = torch.tensor([100.3, 77.7, 20., 10., 0.3, 2., 1.])
    label[3, 2] = torch.tensor([101.9, 78.1, 44., 30., -2.9, 5., 0.])
    label[4, 7] = torch.tensor([200., 20., 12., 24., 3.0, 0., 0.])
    label[1, :6, 4] = torch.tensor([np.pi / 12, -np.pi / 12, 3 * np.pi / 12, 11 * np.pi / 12, -7.0, 9.9])
    return label


def _targets(label):
    B, K = label.shape[:2]
    tgt = torch.empty(B, 10, 64, 64, device=DEV)
    count = torch.full((1,), 99, dtype=torch.int32, device=DEV)      # the entry point clears it
    _call('tfb_centernet_targets', label, B, K, tgt, 64, 64, RATIO, RATIO, 12, count)
    return tgt, count


def _check_targets(tgt, count, label):
    want, avg = O.centernet_targets(label.cpu(), O.Cfg)
    tgt = tgt.cpu()
    assert max(1, int(count)) == avg
    assert torch.allclose(tgt[:, 0:1], want['heat'], rtol=0, atol=1e-6) and torch.equal(tgt[:, 0:1] == 1, want['heat'] == 1)
    assert torch.equal(tgt[:, 1:3], want['wh']) and torch.equal(tgt[:, 3:5], want['offset'])
    assert torch.allclose(tgt[:, 5:6], want['yaw_res'], rtol=0, atol=1e-6)
    assert torch.equal(tgt[:, 6:7], want['velocity']) and torch.equal(tgt[:, 7], want['weight'][:, 0])
    assert torch.equal(tgt[:, 8].long(), want['yaw_cls']) and torch.equal(tgt[:, 9].long(), want['brake'])


def _preds(tgt, seed):
    """pred [B, 64, 64, 21]. At every other occupied cell the wh / offset / velocity residuals are exactly 0; at every occupied cell the
    yaw residual sits on or next to the SmoothL1 branch point |d| = 1."""
    B = tgt.shape[0]
    g = _gen(seed)
    p = torch.randn(B, 64, 64, 21, generator=g) * 2
    p[..., 0] = (torch.randn(B, 64, 64, generator=g) * 3).clamp(-12, 12)
    tc = tgt.cpu().permute(0, 2, 3, 1)
    steps = (-1.0, 1.0, 1.0 - 2 ** -20, -(1.0 + 2 ** -20), 0.5, -1.5)
    for j, (b, y, x) in enumerate((tc[..., 7] == 1).nonzero().tolist()):
        if j % 2 == 0:
            p[b, y, x, 1:5], p[b, y, x, 18] = tc[b, y, x, 1:5], tc[b, y, x, 6]
        p[b, y, x, 17] = tc[b, y, x, 5] + steps[j % len(steps)]
    return p


def _oracle(pred, label, dtype):
    """O.centernet_losses evaluated in `dtype` on the fp32 inputs: the seven losses and d(sum_k GOUT[k] * loss_k) / dpred."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        p = pred.detach().cpu().to(dtype).requires_grad_()
        n = p.permute(0, 3, 1, 2)
        preds = [n[:, 0:1].sigmoid(), n[:, 1:3], n[:, 3:5], n[:, 5:17], n[:, 17:18], n[:, 18:19], n[:, 19:21]]
        out = O.centernet_losses(preds, label.cpu(), O.Cfg)
        vals = torch.stack([out[name] for name, _, _ in HEAD])
        (d,) = torch.autograd.grad((vals * torch.tensor(GOUT, dtype=dtype)).sum(), p)
    finally:
        torch.set_default_dtype(old)
    return vals.detach(), d


def _check_centernet(pred, label, tgt, count, ref_dtype=torch.float64):
    """Forward (raw entry point, run twice, and ops.CenterNetLossFn) and backward against the oracle, term by term and per column group."""
    from transfuser_b200 import ops
    B = pred.shape[0]
    pred = pred.to(DEV)
    acc, out7 = torch.empty(7, dtype=torch.float64, device=DEV), torch.empty(7, device=DEV)
    _twice('tfb_centernet_loss_fwd', (pred, tgt, B, 64 * 64, count, acc, out7), acc)
    pm = pred.clone().requires_grad_()
    out = ops.CenterNetLossFn.apply(pm, label, RATIO, RATIO, 12)
    assert torch.equal(out.detach(), out7)
    (d,) = torch.autograd.grad(out, pm, torch.tensor(GOUT, device=DEV))
    ref, d_ref = _oracle(pred, label, ref_dtype)
    ref32 = _oracle(pred, label, torch.float32)[0] if ref_dtype == torch.float64 else ref
    for kk, (name, _, _) in enumerate(HEAD):
        _check_total(out[kk], ref[kk], ref32[kk], name)
    avg = max(1, int(count))
    tc = tgt.cpu().double()
    wt = tc[:, 7, :, :, None]
    wsum = wt.sum(0, keepdim=True)                    # the CE terms' batch-summed weight (the reference's (B,B,H,W) broadcast)
    x = pred[..., 0:1].cpu().double()
    for kk, (name, lo, hi) in enumerate(HEAD):
        coef = GOUT[kk] * LW[kk] / (avg * DIV[kk])
        w = (2 + x.abs()) if kk == 0 else wsum if kk in (3, 6) else wt
        _check_grad(d[..., lo:hi], d_ref[..., lo:hi], 1e-6 * abs(coef) * w, 'd' + name)
    return out, d


@pytest.mark.parametrize('kind', ['empty', 'random', 'border', 'coincident', 'shared'])
@pytest.mark.parametrize('B', [1, 2, 10])
def test_centernet_losses(B, kind):
    """tfb_centernet_targets, then the seven head losses forward and backward, on 64x64 maps. No boxes: count 0 (avg 1), and the six
    regression / classification terms and their gradients are exactly 0."""
    label = _labels(kind, B, 31 * B + len(kind)).to(DEV)
    tgt, count = _targets(label)
    _check_targets(tgt, count, label)
    out, d = _check_centernet(_preds(tgt, B + len(kind)), label, tgt, count)
    if kind == 'empty':
        assert int(count) == 0
        assert (out[1:] == 0).all() and (d[..., 1:] == 0).all()


@pytest.mark.parametrize('regime', ['confident', 'shifted'])
def test_centernet_classification_terms_confident(regime):
    """The yaw-class and brake CE terms on logits that favour the target class by 9, and the same shifted by +1000."""
    B = 2
    label = _labels('random', B, 77).to(DEV)
    tgt, count = _targets(label)
    p = _preds(tgt, 78)
    tc = tgt.cpu()
    cls, brk = tc[:, 8].long(), tc[:, 9].long()
    p[..., 5:17] = torch.randn(B, 64, 64, 12, generator=_gen(79)) + 9.0 * F.one_hot(cls, 12)
    p[..., 19:21] = torch.randn(B, 64, 64, 2, generator=_gen(80)) + 9.0 * F.one_hot(brk, 2)
    if regime == 'shifted':
        p[..., 5:17] += 1000.0
        p[..., 19:21] += 1000.0
    _check_centernet(p, label, tgt, count)


def test_centernet_saturated_heatmap_logits():
    """Heatmap logits with 20 <= |x| <= 40, where sigmoid is 1 in fp32 and the eps-regularised logs of the focal loss differ between
    fp32 and fp64: the reference is the oracle's own fp32 evaluation."""
    B = 2
    label = _labels('random', B, 51).to(DEV)
    tgt, count = _targets(label)
    p = _preds(tgt, 52)
    g = _gen(53)
    p[..., 0] = (torch.rand(B, 64, 64, generator=g) * 20 + 20) * torch.where(torch.rand(B, 64, 64, generator=g) < 0.5, -1.0, 1.0)
    p[..., 0][tgt.cpu()[:, 0] == 1] = torch.tensor([30.0, -30.0, 20.5, -25.0]).repeat(40)[:int((tgt[:, 0] == 1).sum())]
    _check_centernet(p, label, tgt, count, ref_dtype=torch.float32)


def test_centernet_targets_edge_cases():
    """tfb_centernet_targets on the device against the oracle: empty samples, 20 boxes, border cells, two boxes in one cell (the later
    box wins the regression targets, the heatmap keeps the maximum), yaw angles on bin boundaries and outside [-pi, pi]; twice, with the
    same bits."""
    label = _edge_labels().to(DEV)
    tgt, count = _targets(label)
    _check_targets(tgt, count, label)
    assert int((tgt[0] != 0).sum()) == 0
    tgt2, count2 = _targets(label)
    assert torch.equal(_bits(tgt2), _bits(tgt)) and int(count2) == int(count)
