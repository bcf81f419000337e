"""SURVEY.md §8(f) rows built after the training hot path: the inference path (`forward_ego` + one-launch CenterNet decode,
model.py:685-731, 376-497) and the GeometricFusionBackbone variant (geometric_fusion.py, BASELINE config 4).

CPU part: drop-in key sets and the host-side box geometry against the verbatim reference's (tests/golden/reference_checks.npz).
GPU part: the new kernels against plain fp32 PyTorch ops / the CPU oracle."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import torch_oracle as O
from oracle.make_golden_reference import GOLD as REF_GOLD

DEV = 'cuda'   # the emulated re-runs (tests/test_widen_emulated.py, tools/emulated_module_checks.py) switch this to 'cpu'


def _sync():
    if DEV == 'cuda':
        torch.cuda.synchronize()


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


# ------------------------------------------------------------------ CPU: host logic and the drop-in contract
def _reference_keys(key):
    g = np.load(REF_GOLD)
    return [(str(n), str(s)) for n, s in zip(g['sd_%s_keys' % key], g['sd_%s_shapes' % key])]


def _keys(module):
    return [(k, 'x'.join(map(str, v.shape))) for k, v in module.state_dict().items()]


def test_geometric_fusion_state_dict_matches_reference():
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    mine = LidarCenterNet(TrainConfig(), 'cpu', 'geometric_fusion', 'regnety_032', 'regnety_032', use_velocity=False)
    assert _keys(mine) == _reference_keys('geometric_fusion')
    # the reference's own GlobalConfig (its attribute values, stored by oracle/make_golden_reference.py) drives the product module
    import json
    import types
    cfg = types.SimpleNamespace(**json.loads(str(np.load(REF_GOLD)['reference_config_json'])))
    LidarCenterNet(cfg, 'cpu', 'geometric_fusion', 'regnety_032', 'regnety_032', use_velocity=False)


def test_latent_tf_state_dict_matches_reference():
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    mine = LidarCenterNet(TrainConfig(), 'cpu', 'latentTF', 'regnety_032', 'regnety_032', use_velocity=False)
    assert _keys(mine) == _reference_keys('latentTF')


def test_bbox_local_metric_matches_reference():
    """model.py:810-842 (host numpy in the reference too) on seeded decoded rows."""
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig
    mine = LidarCenterNet(TrainConfig(), 'cpu', 'late_fusion', 'regnety_032', 'regnety_032', use_velocity=False)
    g = np.load(REF_GOLD)
    for row, a, ab, ac in zip(g['bbox_rows'], g['bbox_metric'], g['bbox_brake'], g['bbox_conf']):
        (b, bb, bc), (c, cb, cc) = mine.get_bbox_local_metric(row), O.bbox_local_metric(row)
        assert np.allclose(a, b, rtol=1e-5, atol=1e-5) and np.allclose(a, c, rtol=1e-5, atol=1e-5)
        assert ab == bb == cb and ac == bc == cc


def test_decode_oracle_properties():
    """Size-independent properties of the decode restatement (runs anywhere): scores sorted, every kept score is a 3x3 peak of
    the heatmap, box centres lie within one cell of the peak cell, yaw in (-pi, pi]."""
    g = torch.Generator().manual_seed(2)
    heat = torch.rand(3, 1, 64, 64, generator=g)
    preds = [heat] + [torch.randn(3, c, 64, 64, generator=g) * 0.3 for c in (2, 2, 12, 1, 1, 2)]
    boxes, labels = O.decode_heatmap(preds, 12)
    assert boxes.shape == (3, 100, 8) and labels.shape == (3, 100) and int(labels.abs().sum()) == 0
    assert bool((boxes[..., 7][:, :-1] >= boxes[..., 7][:, 1:]).all())
    assert bool((boxes[..., 4] <= np.pi).all()) and bool((boxes[..., 4] > -np.pi - 1e-6).all())
    hmax = F.max_pool2d(heat, 3, 1, 1)
    for b in range(3):
        for r in boxes[b][:10]:
            x, y = int(torch.floor(r[0] / 4 + 0.5).clamp(0, 63)), int(torch.floor(r[1] / 4 + 0.5).clamp(0, 63))
            win = heat[b, 0, max(y - 2, 0):y + 3, max(x - 2, 0):x + 3]
            assert bool((win == r[7]).any()) and bool((hmax[b, 0] == r[7]).any())


# ------------------------------------------------------------------ GPU: new kernels
def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize('shape,grid', [((2, 72, 40, 176), (5, 22)), ((2, 216, 32, 32), (8, 8)), ((1, 1512, 5, 22), (5, 22)), ((2, 6, 16, 24), (4, 3))])
def test_avgpool_grid_matches_torch(shape, grid):
    from transfuser_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(*shape, device=DEV, generator=g, requires_grad=True)
    xm = _nhwc(x.detach()).requires_grad_()
    want = F.adaptive_avg_pool2d(x, grid)
    got = ops.avgpool_grid(xm, *grid)
    assert rel(got.permute(0, 3, 1, 2), want) < 1e-6
    go = torch.randn(*want.shape, device=DEV, generator=g)
    gw, = torch.autograd.grad(want, x, go)
    gm, = torch.autograd.grad(got, xm, _nhwc(go))
    assert rel(gm.permute(0, 3, 1, 2), gw) < 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize('B,hw,HW,C', [(2, (5, 22), (8, 8), 512), (3, (8, 8), (5, 22), 512), (1, (4, 4), (2, 3), 8)])
def test_gather_sum_matches_torch_index(B, hw, HW, C):
    """The reference's B x B advanced index + diagonal + sum (geometric_fusion.py:145-148), including repeated and all-zero
    correspondences (data.py:636-637 pads with index 0)."""
    from transfuser_b200 import ops
    g = torch.Generator().manual_seed(B * 7 + C)
    emb = torch.randn(B, C, *hw, generator=g).to(DEV).requires_grad_()
    pts = torch.stack((torch.randint(0, hw[1], (B, *HW, 5), generator=g), torch.randint(0, hw[0], (B, *HW, 5), generator=g)), -1)
    pts[:, 0, 0] = 0
    pts = pts.to(DEV)
    flat = pts.view(-1, 2)
    t = emb.permute(0, 2, 3, 1).contiguous()[:, flat[:, 1], flat[:, 0]].view(B, B, *HW, 5, -1)
    want = torch.diagonal(t, 0).permute(4, 3, 0, 1, 2).contiguous().sum(-1)                     # [B, C, H, W]
    em = _nhwc(emb.detach()).requires_grad_()
    got = ops.gather_sum(em, pts)
    assert rel(got.permute(0, 3, 1, 2), want) < 1e-6
    go = torch.randn(*want.shape, generator=g).to(DEV)
    gw, = torch.autograd.grad(want, emb, go)
    gm, = torch.autograd.grad(got, em, _nhwc(go))
    assert rel(gm.permute(0, 3, 1, 2), gw) < 1e-5


def _decode_case(case, g):
    B = 2
    heat_logit = torch.randn(B, 1, 64, 64, generator=g) * 2
    if case == 1:
        heat_logit = (heat_logit * 2).round() / 2          # plateaus: equal neighbours all survive the peak test
    if case == 2:
        heat_logit = heat_logit - 8 * (torch.rand(B, 1, 64, 64, generator=g) < 0.999)   # only a handful of confident peaks
    if case == 3:
        heat_logit[:, :, 0, :] = 30.0                       # saturated (sigmoid == 1.0) border row
    rest = [torch.randn(B, c, 64, 64, generator=g) for c in (2, 2, 12, 1, 1, 2)]
    return heat_logit, rest


@pytest.mark.gpu
@pytest.mark.parametrize('case', [0, 1, 2, 3])
def test_centernet_decode_matches_oracle(case):
    """One-launch decode vs oracle.decode_heatmap (pinned to model.py:376-497 in tests/test_oracle.py; stable=True fixes the
    order torch.topk leaves open for equal scores to the kernel's rule). Labels exact; floats within 1e-5 (sigmoid rounding)."""
    from transfuser_b200 import ops
    g = torch.Generator().manual_seed(40 + case)
    heat_logit, rest = _decode_case(case, g)
    want, want_labels = O.decode_heatmap([heat_logit.sigmoid()] + rest, 12, stable=True)
    raw = torch.cat([heat_logit] + rest, dim=1)
    got, got_labels = ops.centernet_decode(_nhwc(raw.to(DEV)), 12, 100, 4.0)
    _sync()
    got, got_labels = got.cpu(), got_labels.cpu()
    assert got.shape == want.shape and torch.equal(got_labels, want_labels)
    assert torch.equal(got[..., 6], want[..., 6])                       # brake class
    assert torch.allclose(got, want, rtol=1e-6, atol=1e-5), (got - want).abs().amax(dim=(0, 1))


def _build(backbone, seed):
    from transfuser_b200 import LidarCenterNet
    from transfuser_b200.config import TrainConfig

    class C(TrainConfig):
        embd_pdrop = attn_pdrop = resid_pdrop = 0.0
    net = LidarCenterNet(C, 'cpu', backbone, 'regnety_032', 'regnety_032', use_velocity=False)
    names = [(n, tuple(p.shape)) for n, p in list(net.named_parameters()) + list(net.named_buffers()) if not n.startswith('_bev')]
    net.load_state_dict(O.deterministic_state(names, seed=seed), strict=False)
    return net, C


@pytest.mark.gpu
def test_geometric_fusion_forward_backward_matches_oracle():
    """BASELINE config 4: the 11 losses vs the fp32 CPU oracle (1e-3 relative, north_star), gradients finite and in the oracle's
    noise band. The product pools before the 1x1 embed and up-samples after the 1x1 deconv (exact reassociations)."""
    net, C = _build('geometric_fusion', 8)
    batch = O.synthetic_batch(2, seed=5)
    batch['bev_points'], batch['cam_points'] = O.synthetic_correspondences(2, seed=5)
    P = {k: v.clone().requires_grad_(v.dtype.is_floating_point and 'running' not in k) for k, v in net.state_dict().items()}
    ref = O.forward(P, batch, O.Cfg, train=True, backbone_name='geometric_fusion')
    w = dict(zip(C.detailed_losses, C.detailed_losses_weights))
    sum(w[k] * ref[k] for k in ref).backward()
    net = net.to(DEV).train()
    cb = {k: v.to(DEV) for k, v in batch.items()}
    out = net(cb['rgb'], cb['lidar'], ego_waypoint=cb['ego_waypoint'], target_point=cb['target_point'],
              target_point_image=cb['target_point_image'], ego_vel=cb['ego_vel'], bev=cb['bev'], label=cb['label'],
              depth=cb['depth'], semantic=cb['semantic'], bev_points=cb['bev_points'], cam_points=cb['cam_points'])
    for k in ref:
        assert abs(out[k].item() - ref[k].item()) <= 1e-3 * max(abs(ref[k].item()), 1e-6), (k, out[k].item(), ref[k].item())
    sum(w[k] * out[k] for k in out).backward()
    named = dict(net.named_parameters())
    e = np.array([rel(p.grad, P[n].grad) for n, p in named.items() if P[n].grad is not None and p.grad is not None])
    print('geometric fusion: median grad rel err vs fp32 oracle %.2e, p95 %.2e' % (np.median(e), np.percentile(e, 95)))
    assert np.median(e) < 5e-2 and all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)
    # scale 4's image branch reads the scale-3 LiDAR embedding (geometric_fusion.py:277), so lidar_conv4 never receives a
    # gradient in the reference; the same parameters (and only those) stay without gradient here
    assert {n for n, p in named.items() if p.grad is None} == {n for n in named if P[n].grad is None} == {
        '_model.lidar_conv4.weight', '_model.lidar_conv4.bias'}


@pytest.mark.gpu
def test_latent_tf_forward_backward_matches_oracle():
    """latentTF.py: same kernels as the TransFuser path, positional grid instead of the LiDAR histogram."""
    net, C = _build('latentTF', 12)
    batch = O.synthetic_batch(2, seed=7)
    P = {k: v.clone().requires_grad_(v.dtype.is_floating_point and 'running' not in k) for k, v in net.state_dict().items()}

    class OC(O.Cfg):
        embd_pdrop = attn_pdrop = resid_pdrop = 0.0
    ref = O.forward(P, batch, OC, train=True, backbone_name='latentTF')
    w = dict(zip(C.detailed_losses, C.detailed_losses_weights))
    sum(w[k] * ref[k] for k in ref).backward()
    net = net.to(DEV).train()
    cb = {k: v.to(DEV) for k, v in batch.items()}
    out = net(cb['rgb'], cb['lidar'], ego_waypoint=cb['ego_waypoint'], target_point=cb['target_point'],
              target_point_image=cb['target_point_image'], ego_vel=cb['ego_vel'], bev=cb['bev'], label=cb['label'],
              depth=cb['depth'], semantic=cb['semantic'])
    for k in ref:
        assert abs(out[k].item() - ref[k].item()) <= 1e-3 * max(abs(ref[k].item()), 1e-6), (k, out[k].item(), ref[k].item())
    sum(w[k] * out[k] for k in out).backward()
    e = np.array([rel(p.grad, P[n].grad) for n, p in net.named_parameters() if not n.endswith('attn.key.bias')])
    print('latentTF: median grad rel err vs fp32 oracle %.2e, p95 %.2e' % (np.median(e), np.percentile(e, 95)))
    assert np.median(e) < 5e-2 and all(torch.isfinite(p.grad).all() for p in net.parameters())


@pytest.mark.gpu
@pytest.mark.parametrize('backbone', ['transFuser', 'late_fusion'])
def test_forward_ego_matches_oracle(backbone):
    """Eval-mode inference (running-stat BatchNorm, no dropout) + decode + host box geometry vs the CPU oracle's forward_ego."""
    net, C = _build(backbone, 9)
    batch = O.synthetic_batch(1, seed=6)
    P = {k: v.clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        want_wp, want_boxes, want_raw = O.forward_ego(P, batch, O.Cfg, backbone_name=backbone)
    net = net.to(DEV).eval()
    cb = {k: v.to(DEV) for k, v in batch.items()}
    wp, boxes = net.forward_ego(cb['rgb'], cb['lidar'], cb['target_point'], cb['target_point_image'], cb['ego_vel'])
    assert rel(wp, want_wp) < 1e-3
    assert len(boxes) == len(want_boxes)
    for (a, ab, ac), (b, bb, bc) in zip(boxes, want_boxes):
        assert np.allclose(a, b, rtol=1e-3, atol=1e-3) and ab == bb and abs(ac - bc) < 1e-4


@pytest.mark.gpu
def test_fused_adamw_matches_torch_adamw_on_device():
    """optim.FusedAdamW (one kernel over the flat buffer, bf16 mirror) vs torch.optim.AdamW on the same gradients, 3 steps."""
    from transfuser_b200 import gemm, optim
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(37, 53), torch.nn.ReLU(), torch.nn.Linear(53, 11)).to(DEV)
    ref = torch.nn.Sequential(torch.nn.Linear(37, 53), torch.nn.ReLU(), torch.nn.Linear(53, 11)).to(DEV)
    ref.load_state_dict(net.state_dict())
    fp = optim.flatten(net)
    gemm.attach_bf16_weights(fp)
    fused = optim.FusedAdamW(net.parameters(), lr=1e-2, weight_decay=1e-2)
    opt = torch.optim.AdamW(ref.parameters(), lr=1e-2, weight_decay=1e-2)
    for step in range(3):
        x = torch.randn(16, 37, device=DEV)
        fused.zero_grad()
        opt.zero_grad()
        net(x).square().mean().backward()
        ref(x).square().mean().backward()
        fused.step()
        opt.step()
        for a, b in zip(net.parameters(), ref.parameters()):
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), (step, (a - b).abs().max())
    assert torch.equal(fp.bf16, fp.flat.bfloat16())
