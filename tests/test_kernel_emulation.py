"""Kernels added for SURVEY.md §8f (decode, geometric-fusion gather / pool, input preparation) and the optimizer / GRU / target
rasterisation kernels of the training step, executed UNCHANGED on the CPU through the emulation in tests/cuda_emul/ (OS threads +
barriers standing in for a thread block; see cuda_emul.h / build_emul.py) by calling their real C-ABI entry points, and
compared with the oracle / plain torch ops. tests/test_ops_emulated.py does the same for every op-level parity test. This is how
indexing and arithmetic were checked in a container without a GPU; the `-m gpu` tests remain the parity tests proper.
Test infrastructure only."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cuda_emul import loader
from oracle import bev_oracle
from oracle import pipeline_oracle as PO
from oracle import torch_oracle as O


def _call(name, *args):
    return loader.emul().call(name, *args)


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize('shape,grid', [((2, 8, 16, 24), (4, 3)), ((1, 6, 10, 44), (5, 22)), ((2, 4, 8, 8), (8, 8))])
def test_avgpool_grid_kernels(shape, grid):
    N, C, H, W = shape
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(1), requires_grad=True)
    want = F.adaptive_avg_pool2d(x, grid)
    xm = _nhwc(x.detach())
    out = torch.empty(N, grid[0], grid[1], C)
    _call('tfb_avgpool_grid_fwd', xm, out, N, H, W, C, grid[0], grid[1])
    assert torch.equal(out.permute(0, 3, 1, 2), want.detach())          # same accumulation order as ATen's CPU kernel
    go = torch.randn(*want.shape, generator=torch.Generator().manual_seed(2))
    gw, = torch.autograd.grad(want, x, go)
    dx = torch.empty(N, H, W, C)
    gon = _nhwc(go)                                    # keep the operand alive across the ctypes call
    _call('tfb_avgpool_grid_bwd', gon, dx, N, H, W, C, grid[0], grid[1], 0)
    assert torch.allclose(dx.permute(0, 3, 1, 2), gw, rtol=0, atol=1e-7)
    base = torch.randn(N, H, W, C, generator=torch.Generator().manual_seed(3))
    acc = base.clone()
    _call('tfb_avgpool_grid_bwd', gon, acc, N, H, W, C, grid[0], grid[1], 1)
    assert torch.allclose(acc, base + dx, rtol=0, atol=1e-6)


@pytest.mark.parametrize('B,hw,HW,C', [(2, (5, 22), (8, 8), 16), (3, (8, 8), (5, 22), 8), (1, (4, 4), (2, 3), 4)])
def test_gather_sum_kernels(B, hw, HW, C):
    g = torch.Generator().manual_seed(B * 7 + C)
    emb = torch.randn(B, C, *hw, generator=g, requires_grad=True)
    pts = torch.stack((torch.randint(0, hw[1], (B, *HW, 5), generator=g), torch.randint(0, hw[0], (B, *HW, 5), generator=g)), -1)
    pts[:, 0, 0] = 0
    pts[0, 0, 1, 0] = torch.tensor([-1, -1])            # python-style negative index = last column / row
    flat = pts.view(-1, 2)
    t = emb.permute(0, 2, 3, 1).contiguous()[:, flat[:, 1], flat[:, 0]].view(B, B, *HW, 5, -1)       # geometric_fusion.py:145
    want = torch.diagonal(t, 0).permute(4, 3, 0, 1, 2).contiguous().sum(-1)
    em = _nhwc(emb.detach())
    out = torch.empty(B, HW[0], HW[1], C)
    _call('tfb_gather_sum_fwd', em, pts, out, B, hw[0], hw[1], C, HW[0] * HW[1], 5)
    assert torch.allclose(out.permute(0, 3, 1, 2), want.detach(), rtol=0, atol=1e-6)
    go = torch.randn(*want.shape, generator=g)
    gw, = torch.autograd.grad(want, emb, go)
    demb = torch.full((B, hw[0], hw[1], C), float('nan'))  # the entry point clears it before the scatter
    gon = _nhwc(go)
    _call('tfb_gather_sum_bwd', gon, pts, demb, B, hw[0], hw[1], C, HW[0] * HW[1], 5)
    assert torch.allclose(demb.permute(0, 3, 1, 2), gw, rtol=1e-5, atol=1e-5)
    # out-of-range correspondences are skipped
    bad = pts.clone()
    bad[0, 0, 0, 0] = torch.tensor([hw[1], 0])
    out2 = torch.empty_like(out)
    _call('tfb_gather_sum_fwd', em, bad, out2, B, hw[0], hw[1], C, HW[0] * HW[1], 5)
    assert torch.allclose(out2[0, 0, 0], out[0, 0, 0] - em[0, pts[0, 0, 0, 0, 1], pts[0, 0, 0, 0, 0]], atol=1e-5)


@pytest.mark.parametrize('case,H,W', [(0, 64, 64), (1, 64, 64), (2, 64, 64), (3, 64, 64), (0, 24, 40)])
def test_centernet_decode_kernel(case, H, W):
    g = torch.Generator().manual_seed(40 + case)
    B = 2
    heat_logit = torch.randn(B, 1, H, W, generator=g) * 2
    if case == 1:
        heat_logit = (heat_logit * 2).round() / 2
    if case == 2:
        heat_logit = heat_logit - 8 * (torch.rand(B, 1, H, W, generator=g) < 0.999)
    if case == 3:
        heat_logit[:, :, 0, :] = 30.0
    rest = [torch.randn(B, c, H, W, generator=g) for c in (2, 2, 12, 1, 1, 2)]
    want, want_labels = O.decode_heatmap([heat_logit.sigmoid()] + rest, 12, stable=True)
    raw = _nhwc(torch.cat([heat_logit] + rest, dim=1))
    boxes = torch.empty(B, 100, 8)
    labels = torch.empty(B, 100, dtype=torch.int32)
    _call('tfb_centernet_decode', raw, B, H, W, 12, 100, 4.0, boxes, labels)
    assert torch.equal(labels.long(), want_labels)
    assert torch.equal(boxes[..., 6], want[..., 6])
    assert torch.allclose(boxes, want, rtol=1e-6, atol=1e-5), (boxes - want).abs().amax(dim=(0, 1))


def test_target_point_kernel():
    pts = [(x, y) for x in (-16.2, -16.0, 15.9, 16.0, 16.1, 0.3) for y in (-1.4, -1.3, 30.6, 30.7, 30.8, 7.77)] + [(1e12, -1e12), (float('nan'), 0.0)]
    tp = torch.tensor(pts, dtype=torch.float64)
    out = torch.empty(len(pts), 1, 256, 256)
    _call('tfb_draw_target_point', tp, len(pts), out)
    for i, p in enumerate(pts):
        assert np.array_equal(out[i].numpy(), PO.draw_target_point(np.array(p)).astype(np.float32)), p


def test_camera_prep_kernel():
    conv = [0, 1, 2, 3, 4, 5, 6, 4, 3, 0, 2, 1, 5, 6, 0, 1, 2, 3, 4, 5, 6, 0, 1]
    H, W, crop = 40, 240, (32, 176)
    fs = [PO.synthetic_frame(s, H=H, W=W) for s in (0, 1, 2)]
    for f, deg in zip(fs, (5.0, -7.9, 0.0)):            # |shift| <= (240 - 176) / 2: the product's host check rejects more
        f['degree'] = deg
    shifts = [int(f['degree'] / 60 * W) for f in fs]
    B = len(fs)
    rgb, depth = (torch.from_numpy(np.stack([f[k] for f in fs])) for k in ('rgb', 'depth'))
    seg = torch.from_numpy(np.stack([f['seg'] for f in fs]))
    lut = torch.zeros(256, dtype=torch.uint8)
    lut[:len(conv)] = torch.tensor(conv, dtype=torch.uint8)
    o_rgb, o_norm = torch.empty(B, 3, *crop), torch.empty(B, *crop, 3)
    o_depth, o_seg = torch.empty(B, *crop), torch.empty(B, *crop, dtype=torch.int64)
    shift_t = torch.tensor(shifts, dtype=torch.int32)
    _call('tfb_camera_prep', rgb, depth, seg, shift_t, lut, B, H, W, crop[0], crop[1], o_rgb, o_norm, o_depth, o_seg)
    for b, f in enumerate(fs):
        c = PO.crop_rgb(f['rgb'], crop, shifts[b])
        assert np.array_equal(o_rgb[b].numpy(), c.astype(np.float32))
        assert np.array_equal(o_norm[b].numpy(), PO.normalize_nhwc(c))
        assert np.array_equal(o_depth[b].numpy(), PO.depth_from_rgb(PO.crop_rgb(f['depth'], crop, shifts[b])).astype(np.float32))
        assert np.array_equal(o_seg[b].numpy(), PO.seg_classes(f['seg'], conv, crop, shifts[b]).astype(np.int64))


def test_aligned_histogram_kernel():
    fs = [PO.synthetic_frame(s, n_points=1500) for s in (0, 1)]
    fs[1]['degree'] = 0.0
    pts = torch.from_numpy(np.stack([f['points'] for f in fs]))
    Ts = [PO.align_transform(f['ego_matrix_0'], f['ego_matrix_1'], f['degree']) for f in fs]
    T = torch.from_numpy(np.stack(Ts)).reshape(2, 16).contiguous()
    n_valid = torch.tensor([1500, 1200], dtype=torch.int32)
    counts = torch.full((2, 2, 256, 256), 7, dtype=torch.int32)    # the entry point clears it before the scatter
    out = torch.empty(2, 2, 256, 256)
    _call('tfb_bev_histogram_aligned', pts, 0, T, n_valid, 2, 1500, counts, out)
    for b, f in enumerate(fs):
        n = int(n_valid[b])
        want = bev_oracle.lidar_to_histogram_features(PO.align_points(f['points'][:n], Ts[b]))
        assert np.array_equal(out[b].numpy(), want)


def test_input_pipeline_host_code_over_emulated_kernels(monkeypatch):
    """transfuser_b200.pipeline.InputPipeline.prepare executed end to end in this container: its three C-ABI calls reach the
    emulated entry points, everything else is the product's own host code."""
    from transfuser_b200 import pipeline
    from transfuser_b200.config import TrainConfig
    lib = loader.patch_product(monkeypatch)
    monkeypatch.setattr(pipeline.InputPipeline, '_require_cuda', lambda self: None)
    conv = [0, 1, 2, 3, 4, 5, 6, 4, 3, 0, 2, 1, 5, 6, 0, 1, 2, 3, 4, 5, 6, 0, 1]
    H, W, crop = 40, 240, (32, 176)
    fs = [PO.synthetic_frame(s, H=H, W=W, n_points=800) for s in (3, 4)]
    for f, deg in zip(fs, (6.0, -3.0)):
        f['degree'] = deg
    raw = dict(rgb=torch.from_numpy(np.stack([f['rgb'] for f in fs])), depth=torch.from_numpy(np.stack([f['depth'] for f in fs])),
               seg=torch.from_numpy(np.stack([f['seg'] for f in fs])),
               crop_shift=torch.tensor([pipeline.crop_shift_pixels(f['degree'], W // 3, 1) for f in fs], dtype=torch.int32),
               points=torch.from_numpy(np.stack([f['points'] for f in fs])),
               transforms=torch.from_numpy(np.stack([pipeline.align_transform(f['ego_matrix_0'], f['ego_matrix_1'], f['degree']) for f in fs])),
               target_point=torch.from_numpy(np.stack([f['target_point'] for f in fs])))
    pipe = pipeline.InputPipeline(TrainConfig(converter=conv), 'cpu', crop=crop)
    out = pipe.prepare(raw)
    assert lib.log == ['tfb_camera_prep', 'tfb_bev_histogram_aligned', 'tfb_draw_target_point']
    for b, f in enumerate(fs):
        shift = int(f['degree'] / 60 * (W // 3))
        T = PO.align_transform(f['ego_matrix_0'], f['ego_matrix_1'], f['degree'])
        assert np.array_equal(out['rgb'][b].numpy(), PO.crop_rgb(f['rgb'], crop, shift).astype(np.float32))
        assert np.array_equal(out['depth'][b].numpy(), PO.depth_from_rgb(PO.crop_rgb(f['depth'], crop, shift)).astype(np.float32))
        assert np.array_equal(out['semantic'][b].numpy(), PO.seg_classes(f['seg'], conv, crop, shift).astype(np.int64))
        assert np.array_equal(out['lidar'][b].numpy(), bev_oracle.lidar_to_histogram_features(PO.align_points(f['points'], T)))
        assert np.array_equal(out['target_point_image'][b].numpy(), PO.draw_target_point(f['target_point']).astype(np.float32))
        assert np.array_equal(out['target_point'][b].numpy(), f['target_point'].astype(np.float32))
    norm = pipe.prepare(raw, normalized_nhwc=True)['rgb']
    assert getattr(norm, '_tfb_nhwc_normalized', False) and norm.shape == (2, crop[0], crop[1], 3)
    assert np.array_equal(norm[0].numpy(), PO.normalize_nhwc(PO.crop_rgb(fs[0]['rgb'], crop, int(fs[0]['degree'] / 60 * (W // 3)))))
    # host-side rejection of a crop that leaves the frame
    bad = dict(raw, crop_shift=torch.tensor([40, 0], dtype=torch.int32))
    with pytest.raises(ValueError):
        pipe.prepare(bad)


def test_autograd_wrappers_over_emulated_kernels(monkeypatch):
    """ops.AvgPoolGridFn / ops.GatherSumFn / ops.centernet_decode (the product's host wrappers: shapes, saved tensors, backward
    plumbing) executed on CPU tensors over the emulated entry points."""
    from transfuser_b200 import ops
    loader.patch_product(monkeypatch)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 8, 16, 24, generator=g, requires_grad=True)
    xm = _nhwc(x.detach()).requires_grad_()
    pts = torch.stack((torch.randint(0, 3, (2, 5, 6, 5), generator=g), torch.randint(0, 4, (2, 5, 6, 5), generator=g)), -1)
    # product composition: pool to a 4x3 grid, gather 5 correspondences per cell of a 5x6 grid
    mine = ops.gather_sum(ops.avgpool_grid(xm, 4, 3), pts)
    pooled = F.adaptive_avg_pool2d(x, (4, 3))
    want = torch.stack([pooled[b].permute(1, 2, 0)[pts[b, ..., 1], pts[b, ..., 0]].sum(2) for b in range(2)])
    assert mine.shape == want.shape == (2, 5, 6, 8) and torch.allclose(mine, want, atol=1e-6)
    go = torch.randn(*want.shape, generator=g)
    gm, = torch.autograd.grad(mine, xm, go)
    gw, = torch.autograd.grad(want, x, go)
    assert torch.allclose(gm.permute(0, 3, 1, 2), gw, atol=1e-5)
    with pytest.raises(RuntimeError):
        ops.gather_sum(xm, pts.int())
    heat = torch.randn(2, 1, 64, 64, generator=g)
    rest = [torch.randn(2, c, 64, 64, generator=g) for c in (2, 2, 12, 1, 1, 2)]
    boxes, labels = ops.centernet_decode(_nhwc(torch.cat([heat] + rest, 1)), 12, 100, 4.0)
    want_boxes, want_labels = O.decode_heatmap([heat.sigmoid()] + rest, 12, stable=True)
    assert labels.dtype == torch.int64 and torch.equal(labels, want_labels) and torch.allclose(boxes, want_boxes, rtol=1e-6, atol=1e-5)
    with pytest.raises(RuntimeError):
        ops.centernet_decode(torch.zeros(1, 64, 64, 20), 12)


def test_centernet_targets_kernel_edge_cases():
    """LidarCenterNetHead.get_targets (model.py:285-374) as rasterised by csrc/losses.cu, against the oracle (itself pinned to
    the reference): empty label sets, the maximum of 20 boxes, boxes on the map border, coincident centres (the later box
    wins the regression targets, the heatmap keeps the maximum), yaw angles on bin boundaries and outside [-pi, pi]."""
    g = torch.Generator().manual_seed(9)
    label = torch.zeros(5, 20, 7)
    r = lambda *s: torch.rand(*s, generator=g)
    label[1, :, 0:2] = r(20, 2) * 253 + 1                      # sample 1: 20 random boxes
    label[1, :, 2:4] = r(20, 2) * 32 + 8
    label[1, :, 4] = r(20) * 2 * np.pi - np.pi
    label[1, :, 5] = r(20) * 8
    label[1, :, 6] = (r(20) < 0.5).float()
    border = torch.tensor([[0.2, 0.3], [255.9, 0.1], [0.4, 255.8], [255.7, 255.9], [128.0, 0.0], [3.99, 251.9]])
    label[2, :6, 0:2] = border                                 # sample 2: centres in the first / last cells
    label[2, :6, 2:4] = torch.tensor([[60., 30.], [8., 8.], [100., 4.], [2., 2.], [16., 90.], [33., 12.]])
    label[2, :6, 4] = torch.tensor([0.0, np.pi, -np.pi, 2 * np.pi / 12, -2 * np.pi / 12 / 2, 7.5])
    label[2, :6, 5] = 1.0
    label[3, 0] = torch.tensor([100.3, 77.7, 20., 10., 0.3, 2., 1.])       # sample 3: two boxes in the same cell + a gap row
    label[3, 2] = torch.tensor([101.9, 78.1, 44., 30., -2.9, 5., 0.])
    label[4, 7] = torch.tensor([200., 20., 12., 24., 3.0, 0., 0.])         # sample 4: a single box after zero rows
    want, avg = O.centernet_targets(label, O.Cfg)
    tgt = torch.empty(5, 10, 64, 64)
    count = torch.full((1,), 99, dtype=torch.int32)                        # the entry point clears it
    _call('tfb_centernet_targets', label, 5, 20, tgt, 64, 64, 64 / 256, 64 / 256, 12, count)
    assert max(1, int(count)) == avg
    assert torch.allclose(tgt[:, 0:1], want['heat'], rtol=0, atol=1e-6) and torch.equal(tgt[:, 0:1] == 1, want['heat'] == 1)
    assert torch.equal(tgt[:, 1:3], want['wh']) and torch.equal(tgt[:, 3:5], want['offset'])
    assert torch.allclose(tgt[:, 5:6], want['yaw_res'], rtol=0, atol=1e-6)
    assert torch.equal(tgt[:, 6:7], want['velocity']) and torch.equal(tgt[:, 7], want['weight'][:, 0])
    assert torch.equal(tgt[:, 8].long(), want['yaw_cls']) and torch.equal(tgt[:, 9].long(), want['brake'])
    assert int((tgt[0] != 0).sum()) == 0


def test_adamw_kernel_matches_torch_adamw():
    """csrc/gru_adamw.cu's fused AdamW vs torch.optim.AdamW over 4 steps (n not a multiple of 4: vector body + scalar tail),
    the bf16 weight mirror (round-to-nearest-even of the updated fp32 value), the device-resident step counter used under
    CUDA-graph replay, gradient scaling (1/world) and the fused zero_grad."""
    n = 1003
    g0 = torch.Generator().manual_seed(0)
    p0 = torch.randn(n, generator=g0)
    ref = p0.clone().requires_grad_()
    opt = torch.optim.AdamW([ref], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    p, m, v = p0.clone(), torch.zeros(n), torch.zeros(n)
    pd, md, vd = p0.clone(), torch.zeros(n), torch.zeros(n)            # second copy driven by the device step counter
    mirror = torch.zeros(n, dtype=torch.bfloat16)
    step_dev = torch.zeros(1, dtype=torch.int32)
    for step in range(1, 5):
        grad = torch.randn(n, generator=g0) * (10.0 ** (step - 3))
        ref.grad = grad.clone()
        opt.step()
        g = (grad * 4).contiguous()                                    # summed over 4 ranks, grad_scale = 1/4
        _call('tfb_adamw_step', p, g, m, v, n, 1e-2, 0.9, 0.999, 1e-8, 1e-2, step, None, 0.25, mirror, 1, None)
        assert int((g != 0).sum()) == 0                                # zero_grad fused
        _call('tfb_step_tick', None, step_dev)
        g2 = (grad * 4).contiguous()
        _call('tfb_adamw_step', pd, g2, md, vd, n, 1e-2, 0.9, 0.999, 1e-8, 1e-2, 0, step_dev, 0.25, None, 0, None)
        assert torch.equal(g2, grad * 4)
        assert torch.allclose(p, ref.detach(), rtol=2e-6, atol=2e-7), (step, (p - ref.detach()).abs().max())
        assert torch.equal(p, pd) and torch.equal(m, md) and torch.equal(v, vd)
        assert torch.equal(mirror, p.bfloat16())
    st = opt.state[ref]
    # torch >= 2.0 updates exp_avg with lerp (m + (g - m)(1 - b1)); the kernel keeps the reference-era b1*m + (1-b1)*g: same value up
    # to fp32 rounding (cancellation when g ~ m). exp_avg_sq uses the same formula on both sides.
    assert torch.allclose(m, st['exp_avg'], rtol=1e-5, atol=1e-7), (m - st['exp_avg']).abs().max()
    assert torch.allclose(v, st['exp_avg_sq'], rtol=2e-6, atol=1e-14), ((v - st['exp_avg_sq']).abs() / st['exp_avg_sq']).max()


def test_gru_kernels_match_torch_gru_rollout():
    """forward_gru (model.py:611-646): 4 autoregressive GRUCell steps + Linear + cumulative sum; forward and full BPTT."""
    torch.manual_seed(5)
    B, steps = 3, 4
    cell, outl = torch.nn.GRUCell(4, 64), torch.nn.Linear(64, 3)
    z0 = torch.randn(B, 64, requires_grad=True)
    tp = torch.randn(B, 2) * 5
    z, x = z0, torch.zeros(B, 2)
    tpn = tp.clone()
    tpn[:, 1] *= -1
    wps = []
    for _ in range(steps):
        z = cell(torch.cat([x, tpn], dim=1), z)
        x = outl(z)[:, :2] + x
        wps.append(x)
    want = torch.stack(wps, dim=1)
    want = torch.cat((want[:, :, :1] - 1.3, want[:, :, 1:]), dim=2)
    ps = [t.detach().contiguous() for t in (cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh, outl.weight, outl.bias)]
    wp, save = torch.empty(B, steps, 2), torch.empty(B, steps, 5 * 64 + 4)
    z0c = z0.detach().contiguous()
    _call('tfb_gru_fwd', z0c, tp, *ps, B, steps, 1.3, wp, save)
    assert torch.allclose(wp, want.detach(), rtol=1e-5, atol=1e-5)
    d = torch.randn(B, steps, 2)
    grads = torch.autograd.grad(want, [z0, cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh, outl.weight, outl.bias], d)
    dz0 = torch.empty(B, 64)
    outs = [torch.full_like(t, float('nan')) for t in ps]             # the entry point clears the parameter gradients
    _call('tfb_gru_bwd', d, save, ps[0], ps[1], ps[4], B, steps, dz0, *outs)
    for a, b, name in zip([dz0] + outs, grads, ('z0', 'w_ih', 'w_hh', 'b_ih', 'b_hh', 'w_out', 'b_out')):
        if name in ('w_out', 'b_out'):
            a, b = a[:2], b[:2]                                         # the third output row never reaches the waypoints
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-5), (name, (a - b).abs().max())


def test_flat_parameter_training_loop_matches_torch(monkeypatch):
    """optim.flatten + ops autograd functions writing gradients straight into the flat buffer + FusedAdamW (with the bf16 weight
    mirror) for three steps, against the same network in plain torch with torch.optim.AdamW — all on CPU over the emulation."""
    from torch import nn
    from transfuser_b200 import gemm, ops, optim
    loader.patch_product(monkeypatch)

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.a, self.ln, self.b = nn.Linear(24, 40), nn.LayerNorm(40), nn.Linear(40, 8, bias=False)
            self.unused = nn.Parameter(torch.ones(5))          # never receives a gradient: must stay untouched, like in torch

        def forward(self, x, mine):
            if mine:
                return ops.linear(ops.layer_norm(ops.linear(x, self.a.weight, self.a.bias, relu=True), self.ln), self.b.weight)
            return self.b(self.ln(F.relu(self.a(x))))

    torch.manual_seed(0)
    net, ref = Net(), Net()
    ref.load_state_dict(net.state_dict())
    fp = optim.flatten(net)
    gemm.attach_bf16_weights(fp)
    fused = optim.FusedAdamW(net.parameters(), lr=5e-3, weight_decay=0.05)
    opt = torch.optim.AdamW(ref.parameters(), lr=5e-3, weight_decay=0.05)
    for step in range(3):
        x = torch.randn(12, 24)
        fused.zero_grad()
        opt.zero_grad()
        l1, l2 = net(x, True).square().mean(), ref(x, False).square().mean()
        assert abs(float(l1) - float(l2)) < 1e-5 * abs(float(l2))
        l1.backward()
        l2.backward()
        # gradients were written in place into the flat buffer (no copies): each .grad is the parameter's flat view
        for p, o in zip(fp.params, fp.offsets):
            assert p.grad is None or p.grad.data_ptr() == fp.grad.data_ptr() + 4 * o
        fused.step()
        opt.step()
        for (n, a), b in zip(net.named_parameters(), ref.parameters()):
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), (step, n, (a - b).abs().max())
    assert torch.equal(net.unused, torch.ones(5)) and torch.equal(ref.unused, torch.ones(5))
    assert torch.equal(fp.bf16, fp.flat.bfloat16())


def test_flat_qkv_pack_gpt_block_training_loop(monkeypatch):
    """optim.FlatParams lays query / key / value weights (and biases) back to back, so ops.AttentionFn runs the three projections,
    their dgrad / wgrad and the bias gradients as one GEMM / reduction each on the [3C, C] pack, writing the gradients straight into
    the pack's span of the flat gradient buffer. Two optimizer steps of the product's GPT Block (transfuser.py:530-549) over the
    emulated kernels against the same block in plain torch + torch.optim.AdamW; then the same with the fusion switched off."""
    from torch import nn
    from transfuser_b200 import ops, optim
    from transfuser_b200.backbone import Block
    lib = loader.patch_product(monkeypatch)
    C, nh, B, T = 24, 4, 2, 9

    def torch_block(blk, x):
        a = blk.attn
        h = F.layer_norm(x, (C,), blk.ln1.weight, blk.ln1.bias, blk.ln1.eps)
        q, k, v = (lin(h).view(B, T, nh, C // nh).transpose(1, 2) for lin in (a.query, a.key, a.value))
        att = F.softmax(q @ k.transpose(-2, -1) / (C // nh) ** 0.5, dim=-1)
        x = x + a.proj((att @ v).transpose(1, 2).reshape(B * T, C))
        h = F.layer_norm(x, (C,), blk.ln2.weight, blk.ln2.bias, blk.ln2.eps)
        return x + blk.mlp[2](F.relu(blk.mlp[0](h)))

    for fused_qkv in (True, False):
        monkeypatch.setattr(ops, 'QKV_FUSED', fused_qkv)
        torch.manual_seed(1)
        net, ref = Block(C, nh, 4, 0.0, 0.0), Block(C, nh, 4, 0.0, 0.0)
        ref.load_state_dict(net.state_dict())
        fp = optim.flatten(net)
        a = net.attn
        off = {id(p): o for p, o in zip(fp.params, fp.offsets)}
        assert off[id(a.key.weight)] == off[id(a.query.weight)] + C * C and off[id(a.value.weight)] == off[id(a.key.weight)] + C * C
        assert off[id(a.key.bias)] == off[id(a.query.bias)] + C and off[id(a.value.bias)] == off[id(a.key.bias)] + C
        assert all(torch.equal(v, ref.state_dict()[k]) for k, v in net.state_dict().items())      # re-homing kept the values
        fused = optim.FusedAdamW(net.parameters(), lr=3e-3, weight_decay=0.05)
        opt = torch.optim.AdamW(ref.parameters(), lr=3e-3, weight_decay=0.05)
        net.train(), ref.train()
        for step in range(2):
            x = torch.randn(B * T, C)
            fused.zero_grad()
            opt.zero_grad()
            lib.log.clear()
            l1, l2 = net.run(x, B, T).square().mean(), torch_block(ref, x).square().mean()
            assert abs(float(l1) - float(l2)) < 1e-5 * abs(float(l2))
            n_fwd = lib.log.count('tfb_gemm_f32_simt')
            l1.backward()
            l2.backward()
            n_all = lib.log.count('tfb_gemm_f32_simt')
            # forward: q|k|v (1 or 3) + scores + AV + proj + 2 MLP; backward: 4 attention products + dgrad/wgrad of q|k|v (2 or 6)
            # + 2 each for proj and the two MLP layers
            assert (n_fwd, n_all - n_fwd) == ((6, 12) if fused_qkv else (8, 16)), (n_fwd, n_all - n_fwd)
            assert lib.log.count('tfb_colsum') == (1 if fused_qkv else 3)       # (Linear bias gradients come out of tfb_grad_prep)
            for p, o in zip(fp.params, fp.offsets):
                assert p.grad is not None and p.grad.data_ptr() == fp.grad.data_ptr() + 4 * o
            for (n, p), q in zip(net.named_parameters(), ref.parameters()):
                tol = 1e-6 + 1e-4 * float(q.grad.abs().max())
                assert torch.allclose(p.grad, q.grad, rtol=1e-4, atol=tol), (step, n, (p.grad - q.grad).abs().max())
            fused.step()
            opt.step()
            for (n, p), q in zip(net.named_parameters(), ref.parameters()):
                if n == 'attn.key.bias':
                    continue        # its true gradient is 0 (softmax shift invariance): Adam normalises the rounding noise to +-lr
                assert torch.allclose(p, q, rtol=1e-4, atol=2e-5), (step, n, (p - q).abs().max())


@pytest.mark.parametrize('dt', [np.float32, np.float64])
def test_bev_histogram_kernel_bit_exact(dt):
    """csrc/bev_hist.cu vs the numpy oracle (bit-identical to data.py:446-470) and the committed reference fixture, including the
    adversarial points on bin edges / the last edge / outside the grid / NaN, empty and single-point clouds, ragged batches."""
    import os
    for seed, n in ((0, 40000), (1, 1000), (3, 64), (4, 1)):
        pts = torch.from_numpy(bev_oracle.synthetic_points(n, seed, dt)[None].copy())
        counts = torch.full((1, 2, 256, 256), 5, dtype=torch.int32)
        out = torch.empty(1, 2, 256, 256)
        _call('tfb_bev_histogram', pts, int(dt is np.float64), None, 1, n, counts, out)
        assert np.array_equal(out[0].numpy(), bev_oracle.lidar_to_histogram_features(pts[0].numpy())), (seed, n)
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'bev_hist.npz'))
    for key in [k for k in g.files if k.startswith('out_%s_' % np.dtype(dt).name)]:
        _, _, seed, n = key.split('_')
        pts = torch.from_numpy(bev_oracle.synthetic_points(int(n), int(seed), dt)[None].copy())
        counts, out = torch.empty(1, 2, 256, 256, dtype=torch.int32), torch.empty(1, 2, 256, 256)
        _call('tfb_bev_histogram', pts, int(dt is np.float64), None, 1, int(n), counts, out)
        assert np.array_equal(out[0].numpy(), g[key]), key
    ns = [3000, 0, 17, 2500]
    batch = np.full((len(ns), 3000, 4), 3.0, dtype=dt)          # padding that WOULD land inside the grid if it were counted
    want = []
    for i, n in enumerate(ns):
        p = bev_oracle.synthetic_points(n, 10 + i, dt) if n else np.zeros((0, 4), dt)
        batch[i, :n] = p
        want.append(bev_oracle.lidar_to_histogram_features(p))
    counts, out = torch.empty(4, 2, 256, 256, dtype=torch.int32), torch.empty(4, 2, 256, 256)
    _call('tfb_bev_histogram', torch.from_numpy(batch), int(dt is np.float64), torch.tensor(ns, dtype=torch.int32), 4, 3000, counts, out)
    assert np.array_equal(out.numpy(), np.stack(want)) and float(out[1].abs().sum()) == 0


@pytest.mark.parametrize('shape', [(128, 64, 32), (70, 72, 72), (33, 200, 100), (1, 64, 50), (20, 3, 64), (129, 65, 17)])
@pytest.mark.parametrize('ta,tb', [(False, True), (False, False), (True, False), (True, True)])
def test_simt_gemm_kernel(shape, ta, tb):
    """csrc/gemm_simt.cu: all four operand layouts with bias, ReLU, alpha and beta, edge tiles, vs an fp64 product."""
    from transfuser_b200 import gemm
    M, N, K = shape
    g = torch.Generator().manual_seed(M * 7 + N)
    a = torch.randn((K, M) if ta else (M, K), generator=g)
    b = torch.randn((N, K) if tb else (K, N), generator=g)
    bias, c0 = torch.randn(N, generator=g), torch.randn(M, N, generator=g)
    out = c0.clone()
    lib = loader.emul()
    import transfuser_b200._lib as L
    old, L._LIB = L._LIB, lib
    try:
        gemm.gemm(a, b, out, ta, tb, bias=bias, relu=True, alpha=0.5, beta=1.0, mode='simt')
        A, B = (a.double().t() if ta else a.double()), (b.double().t() if tb else b.double())
        want = (0.5 * (A @ B) + bias.double() + c0.double()).clamp_min(0)
        assert ((out.double() - want).norm() / want.norm()).item() < 1e-6
        # strided views: a column window of x as A, a column window of the output as C (the packed q|k|v layout)
        x, w = torch.randn(40, 3 * 24, generator=g), torch.randn(24, 24, generator=g)
        dst = torch.zeros(40, 3 * 24)
        gemm.gemm(x[:, 24:48], w, dst[:, 48:], False, True, mode='simt')
        assert torch.allclose(dst[:, 48:].double(), x[:, 24:48].double() @ w.double().t(), atol=1e-5) and float(dst[:, :48].abs().sum()) == 0
    finally:
        L._LIB = old


def test_conv3x3_weight_pack_batched_matches_single_pack():
    """tfb_conv3x3_pack_weights_batched (every registered conv of the model in one launch, device-resident descriptor table) writes
    exactly what per-conv tfb_conv3x3_pack_weights calls write, for the dense / grouped, forward / dgrad plans of ops._conv_tc_plan;
    the single pack itself is checked against the layout definition (conv_pack.cu) restated in numpy."""
    from transfuser_b200 import ops
    cases = [(64, 64, 1), (32, 32, 1), (512, 128, 1), (72, 72, 3), (216, 216, 9), (128, 64, 1), (32, 7 + 1, 1)]
    rows, keep, singles = [], [], []
    for n, (cin, cout, groups) in enumerate(cases):
        w = torch.randn(cout, cin // groups, 3, 3, generator=torch.Generator().manual_seed(n))
        for mode in (0, 1):
            c_read, c_write = (cin, cout) if mode == 0 else (cout, cin)
            plan = ops._conv_tc_plan(c_read, c_write, groups)
            if plan is None:
                continue
            shape = (plan['gblocks'], plan['nchunks'], 9, plan['NB'], plan['KC'])
            args = (cout, cin, groups, mode, plan['NB'], plan['KC'], plan['c_step'], plan['nchunks'], plan['nb_real'], plan['gblocks'])
            one = torch.full(shape, 7.0, dtype=torch.bfloat16)
            _call('tfb_conv3x3_pack_weights', w, one, *args)
            many = torch.full(shape, 9.0, dtype=torch.bfloat16)
            rows.append([w.data_ptr(), many.data_ptr()] + list(args))
            keep.append((w, many))
            singles.append(one)
            # layout definition, restated
            want = np.zeros(shape, np.float32)
            wn = w.numpy()
            cig, cog = cin // groups, cout // groups
            for gb in range(shape[0]):
                for ch in range(shape[1]):
                    for j in range(min(plan['nb_real'], shape[3])):
                        oc = gb * plan['nb_real'] + j
                        for kk in range(shape[4]):
                            rc = gb * plan['c_step'] + ch * plan['KC'] + kk
                            if mode == 0 and oc < cout and rc < cin and rc // cig == oc // cog:
                                want[gb, ch, :, j, kk] = wn[oc, rc - (oc // cog) * cig].reshape(9)
                            if mode == 1 and oc < cin and rc < cout and rc // cog == oc // cig:
                                want[gb, ch, :, j, kk] = wn[rc, oc - (oc // cig) * cig].reshape(9)[::-1]
            assert torch.equal(one.float(), torch.from_numpy(want).bfloat16().float()), (cin, cout, groups, mode)
    table = torch.tensor(rows, dtype=torch.int64)
    _call('tfb_conv3x3_pack_weights_batched', table, len(rows), 3)
    assert len(rows) >= 10
    for (w, many), one in zip(keep, singles):
        assert torch.equal(many.view(torch.int16), one.view(torch.int16))


@pytest.mark.parametrize('N,H,W,C,groups,stride', [(2, 6, 7, 48, 2, 1), (1, 9, 8, 72, 3, 2), (2, 5, 4, 64, 1, 1), (1, 4, 6, 32, 1, 2),
                                                    (1, 3, 3, 216, 9, 1)])
def test_im2col_channel_tap_order(N, H, W, C, groups, stride):
    """tfb_im2col3x3_bf16 writes col[m][c][tap] (tap fastest) = F.unfold's channel-major patch order, i.e. the order of PyTorch's
    weight layout [co][ci][kh][kw]: dW = dy^T col then IS the weight gradient, no permute pass. Checked bit-exactly (bf16 rounding
    of the same fp32 values), zero padding at the borders included, and through the implied fp32 GEMM against torch's conv wgrad."""
    g = torch.Generator().manual_seed(N * 100 + C)
    x = torch.randn(N, C, H, W, generator=g)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    col = torch.full((N * Ho * Wo, 9 * C), 3.0, dtype=torch.bfloat16)
    xm = _nhwc(x)
    _call('tfb_im2col3x3_bf16', xm, col, N, H, W, C, stride, groups)
    want = F.unfold(x, 3, padding=1, stride=stride).permute(0, 2, 1).reshape(N * Ho * Wo, 9 * C).bfloat16()
    assert torch.equal(col.view(torch.int16), want.view(torch.int16))
    # dW_g = dy_g^T col_g in PyTorch layout
    Cout = 2 * groups * 4
    w = torch.randn(Cout, C // groups, 3, 3, generator=g, requires_grad=True)
    xb = x.bfloat16().float()
    y = F.conv2d(xb, w, None, stride=stride, padding=1, groups=groups)
    dy = torch.randn(y.shape, generator=g)
    gw, = torch.autograd.grad(y, w, dy)
    dym = dy.permute(0, 2, 3, 1).reshape(-1, Cout)
    Cig, Cog = C // groups, Cout // groups
    got = torch.cat([dym[:, k * Cog:(k + 1) * Cog].t() @ col.float()[:, k * 9 * Cig:(k + 1) * 9 * Cig] for k in range(groups)])
    assert torch.allclose(got.view(Cout, Cig, 3, 3), gw, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize('M,Cin,Cout,bias', [(4100, 64, 1, False), (4099, 64, 12, True), (700, 72, 3, True), (517, 130, 16, False), (33, 8, 2, True)])
def test_conv1x1_wgrad_narrow_output_kernel(M, Cin, Cout, bias):
    """tfb_conv2d_wgrad, k = 1, Cout <= 16 (the CenterNet head outputs 64 -> {1, 2, 3, 12}): threads over input channels, dy broadcast,
    register accumulators — dW = dy^T x and dbias = column sums of dy against torch, ragged pixel counts / channel blocks included."""
    g = torch.Generator().manual_seed(M + Cout)
    x, dy = torch.randn(M, Cin, generator=g), torch.randn(M, Cout, generator=g)
    dw = torch.full((Cout, Cin), float('nan'))
    db = torch.full((Cout,), float('nan')) if bias else None
    _call('tfb_conv2d_wgrad', x, dy, dw, db, 1, M, 1, Cin, Cout, 1, 1, 1)
    want = dy.double().t() @ x.double()
    assert torch.allclose(dw.double(), want, rtol=1e-4, atol=1e-4 * float(want.abs().max()))
    if bias:
        assert torch.allclose(db.double(), dy.double().sum(0), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize('H,W,gh,gw,C', [(40, 176, 5, 22, 8), (37, 50, 5, 22, 4), (5, 22, 5, 22, 8), (16, 16, 8, 8, 12), (3, 9, 8, 8, 4)])
def test_gpt_up_add_backward_gather(H, W, gh, gw, C):
    """tfb_gpt_up_add_bwd as a gather (no atomics, no zero fill): every element of its token range is written exactly once (NaN-filled
    destination), the rest of dtok is untouched, and the values equal autograd through F.interpolate on the view-quirk slab — also
    for non-integer scales and for a feature map smaller than the anchor grid."""
    N, T, t_off = 2, gh * gw + 7, 3
    g = torch.Generator().manual_seed(H * W)
    dy = torch.randn(N, H, W, C, generator=g)
    dtok = torch.full((N, T, C), float('nan'))
    _call('tfb_gpt_up_add_bwd', dy, dtok, N, H, W, C, gh, gw, t_off, T)
    slab = torch.zeros(N, C, gh, gw, requires_grad=True)          # the (C, gh, gw) view of the token slab (transfuser.py:363-364)
    up = F.interpolate(slab, size=(H, W), mode='bilinear', align_corners=False)
    want, = torch.autograd.grad(up, slab, dy.permute(0, 3, 1, 2))
    got = dtok[:, t_off:t_off + gh * gw].reshape(N, C, gh, gw)     # same memory re-interpretation as the reference's .view
    assert torch.isfinite(got).all()
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-5)
    assert torch.isnan(dtok[:, :t_off]).all() and torch.isnan(dtok[:, t_off + gh * gw:]).all()


@pytest.mark.parametrize('Hi,Wi,Ho,Wo,C,ac', [(5, 22, 40, 176, 4, 0), (8, 8, 16, 16, 8, 0), (64, 64, 160, 160, 2, 1), (7, 5, 19, 23, 3, 0),
                                              (7, 5, 19, 23, 3, 1), (6, 6, 6, 6, 4, 1), (9, 9, 4, 5, 4, 0), (4, 4, 1, 1, 4, 1), (2, 3, 40, 50, 3, 0), (2, 3, 40, 50, 3, 1),
                                              (3, 3, 28, 28, 4, 1)])
def test_upsample_bilinear_backward_gather(Hi, Wi, Ho, Wo, C, ac):
    """tfb_upsample_bilinear_bwd as a gather (no atomics, no memset): dx written exactly once (NaN-filled destination) and equal to
    autograd through F.interpolate — integer / fractional scales, align_corners on and off, identity and down-sampling sizes."""
    N = 2
    g = torch.Generator().manual_seed(Hi * Wo + ac)
    dy = torch.randn(N, Ho, Wo, C, generator=g)
    dx = torch.full((N, Hi, Wi, C), float('nan'))
    _call('tfb_upsample_bilinear_bwd', dy, dx, N, Hi, Wi, Ho, Wo, C, ac)
    x = torch.zeros(N, C, Hi, Wi, requires_grad=True)
    want, = torch.autograd.grad(F.interpolate(x, size=(Ho, Wo), mode='bilinear', align_corners=bool(ac)), x, dy.permute(0, 3, 1, 2))
    assert torch.isfinite(dx).all()
    assert torch.allclose(dx.permute(0, 3, 1, 2), want, rtol=1e-5, atol=1e-5)
